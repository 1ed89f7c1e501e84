// actnn.cu -- activation-compressed training (ActNN) for sm_90a: group min/max, quantize + bit-pack, unpack +
// dequantize, 1-bit ReLU / dropout masks and the per-row bit allocation.
//
// Quantization of an [N, D] fp32 activation (D zero-padded to Dp, a multiple of the group size gs = 64 | 256;
// G = Dp / gs groups per row).  Per group: mn, mx over its gs values (padding included, as the reference pads before
// its minimax), then with B = 2^b - 1 (b = the row's bit width)
//     mn' = mn - 1e-6f,  mx' = mx + 1e-6f,  scale = B / (mx' - mn')
//     v = (x - mn') * scale  [+ u - 0.5f, u = (draw(seed, n * Dp + d, 0) >> 40) * 2^-24, when stochastic]
//     q = rint(min(max(v, 0), B))
// in fp32 with no contraction: the reference's torch path (actnn/ops.py:22-41, quantize_and_pack with
// config.simulate), whose codes are those of its pack kernels with the noise at 0.5.  scale and mn are kept as bf16
// (ops.py:115-116); the dequantized value is q / scale_bf16 + mn_bf16 (ops.py:55-57).
//
// Packed layout (ours, not the reference's bytes): row n is a bitstream of Dp codes of b_n bits, code d at bits
// [d * b_n, (d + 1) * b_n), LSB first in little-endian bytes; it starts at byte row_off[n] (mixed widths: an exclusive
// prefix sum of b * Dp / 8) or n * Dp * b / 8 (one width).  Eight codes are b bytes, so each thread owns 8 codes and
// writes whole bytes; a group of gs codes is gs / 8 lanes of one warp, which reduce its min / max with shuffles.
//
// Masks (QReLU, QDropout): bit i of 32-bit word i / 32 is element i (a __ballot_sync per warp).  The dropout keeps
// element i iff draw(seed, i, 0) >= drop_below = floor(p * 2^64) and scales a kept value by 1 / (1 - p) in double,
// as the reference's kernel does (quantization_cuda_kernel.cu:540, :601).
//
// Bit allocation (cogdl_b200_actnn_bits): the reference greedy (calc_precision.cc:9-50, w = 1) decrements the row of
// the largest key (float)(C_i * (1 / (2^b - 1)^2 - 1 / (2^(b-1) - 1)^2)) in priority_queue<pair<float, int64_t>>
// order until sum(b) <= target.  For C_i >= 0 a row's keys fall (weakly) as b falls, so the greedy pops the keys of
// all rows in one descending order and the result is a top-K selection: K = b0 * N - target keys out of the
// (b0 - 1) * N keys (b = b0 .. 2), and b_i = b0 - (selected keys of row i).  Each key is made unique as the 64-bit
// (order-preserving float bits << 32 | i << 3 | b - 1): ties in the float order go to the larger row, as in the
// pair order, and within a row to the larger b, the order the greedy pushes them.  The keys are radix-sorted on the
// device, the K-th largest is the threshold and each row counts its keys at or above it.
#include <cuda_bf16.h>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "rng.cuh"

namespace cogdl_b200 {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float stochastic_noise(uint64_t seed, int64_t flat) {
  return __fsub_rn(__uint2float_rn((uint32_t)(draw(seed, flat, 0) >> 40)) * 0x1p-24f, 0.5f);
}

// One thread = 8 consecutive codes of one row.  MODE 0: group min / max only; MODE 1: quantize and pack;
// MODE 2: unpack and dequantize.
template <int MODE, int GS>
__global__ void __launch_bounds__(kThreads) actnn_group_kernel(
    const float *__restrict__ x, int64_t N, int64_t D, int64_t Dp, const int32_t *__restrict__ bits, int uniform_bits,
    const int64_t *__restrict__ row_off, int stochastic, uint64_t seed, float *__restrict__ mn_out,
    float *__restrict__ mx_out, uint8_t *__restrict__ packed, const uint8_t *__restrict__ packed_in,
    __nv_bfloat16 *__restrict__ scale_out, __nv_bfloat16 *__restrict__ mnq_out,
    const __nv_bfloat16 *__restrict__ scale_in, const __nv_bfloat16 *__restrict__ mnq_in, float *__restrict__ out) {
  constexpr int L = GS / 8;   // lanes per group
  const int64_t oct_per_row = Dp / 8;
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const bool active = t < N * oct_per_row;
  const int64_t n = active ? t / oct_per_row : 0;
  const int64_t o = active ? t - n * oct_per_row : 0;   // octet within the row
  const int64_t d0 = o * 8;                              // first padded column
  const int64_t grp = n * (Dp / GS) + d0 / GS;           // group index in [N * G]
  const int lane_in_group = (int)(o % L);
  const int b = active ? (bits ? bits[n] : uniform_bits) : 1;
  const int64_t base = active ? (bits ? row_off[n] : n * oct_per_row * b) : 0;

  if (MODE == 2) {
    if (!active) return;
    uint64_t w = 0;
    const uint8_t *src = packed_in + base + o * b;
    for (int k = 0; k < b; ++k) w |= (uint64_t)src[k] << (8 * k);
    const float s = __bfloat162float(scale_in[grp]);
    const float m = __bfloat162float(mnq_in[grp]);
    const uint64_t cmask = (1ull << b) - 1;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int64_t d = d0 + k;
      if (d < D) {
        const float q = (float)((w >> (k * b)) & cmask);
        out[n * D + d] = __fadd_rn(__fdiv_rn(q, s), m);
      }
    }
    return;
  }

  float v[8];
  float lo = INFINITY, hi = -INFINITY;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int64_t d = d0 + k;
    v[k] = (active && d < D) ? __ldg(x + n * D + d) : 0.f;
    lo = fminf(lo, v[k]);
    hi = fmaxf(hi, v[k]);
  }
#pragma unroll
  for (int s = L / 2; s > 0; s >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(FULL, lo, s));
    hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, s));
  }
  if (!active) return;
  if (MODE == 0) {
    if (lane_in_group == 0) {
      mn_out[grp] = lo;
      mx_out[grp] = hi;
    }
    return;
  }
  const float B = (float)((1 << b) - 1);
  const float mnp = __fsub_rn(lo, 1e-6f), mxp = __fadd_rn(hi, 1e-6f);
  const float scale = __fdiv_rn(B, __fsub_rn(mxp, mnp));
  if (lane_in_group == 0) {
    scale_out[grp] = __float2bfloat16_rn(scale);
    mnq_out[grp] = __float2bfloat16_rn(lo);
  }
  uint64_t w = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    float y = __fmul_rn(__fsub_rn(v[k], mnp), scale);
    if (stochastic) y = __fadd_rn(y, stochastic_noise(seed, n * Dp + d0 + k));
    y = rintf(fminf(fmaxf(y, 0.f), B));
    w |= (uint64_t)(uint32_t)y << (k * b);
  }
  // 8 codes = b bytes at a b-aligned offset (row starts are multiples of 8 bytes)
  uint8_t *dst = packed + base + o * b;
  switch (b) {
    case 1: *dst = (uint8_t)w; break;
    case 2: *reinterpret_cast<uint16_t *>(dst) = (uint16_t)w; break;
    case 4: *reinterpret_cast<uint32_t *>(dst) = (uint32_t)w; break;
    case 8: *reinterpret_cast<uint64_t *>(dst) = w; break;
    default:
      for (int k = 0; k < b; ++k) dst[k] = (uint8_t)(w >> (8 * k));
  }
}

// MODE 0: relu forward (y = x > 0 ? x : 0, bit = x > 0); MODE 1: dropout forward (bit = keep, y = x / (1 - p)).
template <int MODE>
__global__ void __launch_bounds__(kThreads) actnn_mask_fwd_kernel(const float *__restrict__ x, int64_t n, double keep_div,
                                                                  uint64_t seed, uint64_t drop_below,
                                                                  float *__restrict__ y, uint32_t *__restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  bool bit = false;
  if (i < n) {
    const float v = x[i];
    if (MODE == 0) {
      bit = v > 0.f;
      y[i] = bit ? v : 0.f;
    } else {
      bit = draw(seed, i, 0) >= drop_below;
      y[i] = bit ? (float)((double)v / keep_div) : 0.f;
    }
  }
  const unsigned word = __ballot_sync(FULL, bit);
  if ((threadIdx.x & 31) == 0 && i < n) mask[i >> 5] = word;
}

// MODE 0: relu backward (gx = bit ? g : 0); MODE 1: dropout backward (gx = bit ? g / (1 - p) : 0).
template <int MODE>
__global__ void __launch_bounds__(kThreads) actnn_mask_bwd_kernel(const float *__restrict__ g,
                                                                  const uint32_t *__restrict__ mask, int64_t n,
                                                                  double keep_div, float *__restrict__ gx) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const bool bit = (__ldg(mask + (i >> 5)) >> (i & 31)) & 1u;
  const float v = g[i];
  gx[i] = bit ? (MODE == 0 ? v : (float)((double)v / keep_div)) : 0.f;
}

// ---------------------------------------------------------------- bit allocation
__device__ __forceinline__ uint64_t alloc_key(float c, int64_t row, int b) {
  const int c1 = ((1 << b) - 1) * ((1 << b) - 1);
  const int c2 = ((1 << (b - 1)) - 1) * ((1 << (b - 1)) - 1);
  float delta = (float)((double)c * (1.0 / c1 - 1.0 / c2));
  if (delta == 0.f) delta = 0.f;   // -0.0 and +0.0 are one key in the float order
  uint32_t u = __float_as_uint(delta);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((uint64_t)u << 32) | ((uint64_t)row << 3) | (uint64_t)(b - 1);
}

__global__ void actnn_alloc_keys_kernel(const float *__restrict__ C, int64_t N, int b0, uint64_t *__restrict__ keys,
                                        int *__restrict__ bad) {
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const int per_row = b0 - 1;
  if (t >= N * per_row) return;
  const int64_t i = t / per_row;
  const int b = b0 - (int)(t - i * per_row);
  const float c = C[i];
  if (!(c >= 0.f) || isinf(c)) *bad = 1;   // NaN, infinite or negative: the greedy is not a top-K there
  keys[t] = alloc_key(c, i, b);
}

__global__ void actnn_alloc_count_kernel(const float *__restrict__ C, int64_t N, int b0, int64_t K,
                                         const uint64_t *__restrict__ sorted, int32_t *__restrict__ bits) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  int taken = 0;
  if (K > 0) {
    const uint64_t thr = sorted[K - 1];
    const float c = C[i];
    for (int b = b0; b >= 2; --b) {
      if (alloc_key(c, i, b) < thr) break;
      ++taken;
    }
  }
  bits[i] = b0 - taken;
}

static int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }

static size_t sort_temp_bytes(int64_t n_keys) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortKeysDescending((void *)nullptr, bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                           (int)(n_keys > 0 ? n_keys : 1));
  return bytes;
}

int check_group(int64_t N, int64_t D, int32_t group_size, const char *who) {
  CB_REQUIRE(N >= 0 && D > 0, "%s: bad shape [%lld, %lld]", who, (long long)N, (long long)D);
  CB_REQUIRE(group_size == 64 || group_size == 256, "%s: group_size must be 64 or 256, got %d", who, group_size);
  return COGDL_B200_OK;
}

template <int MODE>
int launch_group(int64_t N, int64_t D, int32_t gs, cudaStream_t s, const char *name, const float *x,
                 const int32_t *bits, int uniform_bits, const int64_t *row_off, int stochastic, uint64_t seed,
                 float *mn, float *mx, uint8_t *packed, const uint8_t *packed_in, __nv_bfloat16 *scale_out,
                 __nv_bfloat16 *mnq_out, const __nv_bfloat16 *scale_in, const __nv_bfloat16 *mnq_in, float *out) {
  const int64_t Dp = ceil_div(D, gs) * gs;
  const int64_t blocks = ceil_div(N * (Dp / 8), kThreads);
  note_kernel("%s<%d>", name, (int)gs);
  if (blocks == 0) return COGDL_B200_OK;
  CB_REQUIRE(blocks <= 0x7fffffffLL, "%s: problem too large for one launch", name);
  auto kernel = gs == 64 ? actnn_group_kernel<MODE, 64> : actnn_group_kernel<MODE, 256>;
  kernel<<<(unsigned)blocks, kThreads, 0, s>>>(x, N, D, Dp, bits, uniform_bits, row_off, stochastic, seed, mn, mx,
                                               packed, packed_in, scale_out, mnq_out, scale_in, mnq_in, out);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

int check_widths(const int32_t *bits, int32_t uniform_bits, const int64_t *row_off, const char *who) {
  if (bits) {
    CB_REQUIRE(row_off != nullptr, "%s: mixed bit widths need row_offsets", who);
  } else {
    CB_REQUIRE(uniform_bits == 1 || uniform_bits == 2 || uniform_bits == 4 || uniform_bits == 8,
               "%s: a uniform bit width must be 1, 2, 4 or 8, got %d", who, uniform_bits);
  }
  return COGDL_B200_OK;
}

}  // namespace
}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int cogdl_b200_actnn_minmax_f32(const float *x, int64_t N, int64_t D, int32_t group_size, float *mn,
                                           float *mx, cogdl_b200_stream_t stream) {
  if (int rc = check_group(N, D, group_size, "actnn_minmax")) return rc;
  CB_REQUIRE(N == 0 || (x && mn && mx), "actnn_minmax: null pointer");
  return launch_group<0>(N, D, group_size, (cudaStream_t)stream, "actnn_minmax", x, nullptr, 1, nullptr, 0, 0, mn, mx,
                         nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int cogdl_b200_actnn_pack_f32(const float *x, int64_t N, int64_t D, int32_t group_size, const int32_t *bits,
                                         int32_t uniform_bits, const int64_t *row_offsets, int32_t stochastic,
                                         uint64_t seed, uint8_t *packed, void *scale_bf16, void *mn_bf16,
                                         cogdl_b200_stream_t stream) {
  if (int rc = check_group(N, D, group_size, "actnn_pack")) return rc;
  if (int rc = check_widths(bits, uniform_bits, row_offsets, "actnn_pack")) return rc;
  CB_REQUIRE(N == 0 || (x && packed && scale_bf16 && mn_bf16), "actnn_pack: null pointer");
  return launch_group<1>(N, D, group_size, (cudaStream_t)stream, bits ? "actnn_pack_mixed" : "actnn_pack", x, bits,
                         uniform_bits, row_offsets, stochastic ? 1 : 0, seed, nullptr, nullptr, packed, nullptr,
                         (__nv_bfloat16 *)scale_bf16, (__nv_bfloat16 *)mn_bf16, nullptr, nullptr, nullptr);
}

extern "C" int cogdl_b200_actnn_unpack_f32(const uint8_t *packed, int64_t N, int64_t D, int32_t group_size,
                                           const int32_t *bits, int32_t uniform_bits, const int64_t *row_offsets,
                                           const void *scale_bf16, const void *mn_bf16, float *out,
                                           cogdl_b200_stream_t stream) {
  if (int rc = check_group(N, D, group_size, "actnn_unpack")) return rc;
  if (int rc = check_widths(bits, uniform_bits, row_offsets, "actnn_unpack")) return rc;
  CB_REQUIRE(N == 0 || (packed && scale_bf16 && mn_bf16 && out), "actnn_unpack: null pointer");
  return launch_group<2>(N, D, group_size, (cudaStream_t)stream, bits ? "actnn_unpack_mixed" : "actnn_unpack",
                         nullptr, bits, uniform_bits, row_offsets, 0, 0, nullptr, nullptr, nullptr, packed, nullptr,
                         nullptr, (const __nv_bfloat16 *)scale_bf16, (const __nv_bfloat16 *)mn_bf16, out);
}

template <int MODE>
static int mask_fwd(const float *x, int64_t n, double keep_div, uint64_t seed, uint64_t drop_below, float *y,
                    uint32_t *mask, cudaStream_t s, const char *name) {
  CB_REQUIRE(n >= 0, "%s: negative size", name);
  CB_REQUIRE(n == 0 || (x && y && mask), "%s: null pointer", name);
  note_kernel("%s", name);
  const int64_t blocks = ceil_div(n, kThreads);
  if (blocks == 0) return COGDL_B200_OK;
  CB_REQUIRE(blocks <= 0x7fffffffLL, "%s: problem too large for one launch", name);
  actnn_mask_fwd_kernel<MODE><<<(unsigned)blocks, kThreads, 0, s>>>(x, n, keep_div, seed, drop_below, y, mask);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

template <int MODE>
static int mask_bwd(const float *g, const uint32_t *mask, int64_t n, double keep_div, float *gx, cudaStream_t s,
                    const char *name) {
  CB_REQUIRE(n >= 0, "%s: negative size", name);
  CB_REQUIRE(n == 0 || (g && mask && gx), "%s: null pointer", name);
  note_kernel("%s", name);
  const int64_t blocks = ceil_div(n, kThreads);
  if (blocks == 0) return COGDL_B200_OK;
  CB_REQUIRE(blocks <= 0x7fffffffLL, "%s: problem too large for one launch", name);
  actnn_mask_bwd_kernel<MODE><<<(unsigned)blocks, kThreads, 0, s>>>(g, mask, n, keep_div, gx);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_actnn_relu_fwd_f32(const float *x, int64_t n, float *y, uint32_t *mask,
                                             cogdl_b200_stream_t stream) {
  return mask_fwd<0>(x, n, 1.0, 0, 0, y, mask, (cudaStream_t)stream, "actnn_relu_fwd");
}

extern "C" int cogdl_b200_actnn_relu_bwd_f32(const float *g, const uint32_t *mask, int64_t n, float *gx,
                                             cogdl_b200_stream_t stream) {
  return mask_bwd<0>(g, mask, n, 1.0, gx, (cudaStream_t)stream, "actnn_relu_bwd");
}

extern "C" int cogdl_b200_actnn_dropout_fwd_f32(const float *x, int64_t n, float p, uint64_t seed,
                                                uint64_t drop_below, float *y, uint32_t *mask,
                                                cogdl_b200_stream_t stream) {
  CB_REQUIRE(p >= 0.f && p < 1.f, "actnn_dropout_fwd: p must be in [0, 1), got %g", (double)p);
  return mask_fwd<1>(x, n, 1.0 - (double)p, seed, drop_below, y, mask, (cudaStream_t)stream, "actnn_dropout_fwd");
}

extern "C" int cogdl_b200_actnn_dropout_bwd_f32(const float *g, const uint32_t *mask, int64_t n, float p, float *gx,
                                                cogdl_b200_stream_t stream) {
  CB_REQUIRE(p >= 0.f && p < 1.f, "actnn_dropout_bwd: p must be in [0, 1), got %g", (double)p);
  return mask_bwd<1>(g, mask, n, 1.0 - (double)p, gx, (cudaStream_t)stream, "actnn_dropout_bwd");
}

extern "C" int64_t cogdl_b200_actnn_bits_scratch_bytes(int64_t N) {
  const int64_t n_keys = 7 * (N > 0 ? N : 1);
  return 256 + 2 * align256(n_keys * 8) + align256((int64_t)sort_temp_bytes(n_keys));
}

extern "C" int cogdl_b200_actnn_bits(const float *C, int64_t N, int32_t initial_bits, int64_t target, int32_t *bits,
                                     void *scratch, int64_t scratch_bytes, cogdl_b200_stream_t stream) {
  CB_REQUIRE(N >= 0 && N < (1LL << 28), "actnn_bits: N must be in [0, 2^28), got %lld", (long long)N);
  CB_REQUIRE(initial_bits >= 1 && initial_bits <= 8, "actnn_bits: initial_bits must be in 1..8, got %d", initial_bits);
  CB_REQUIRE(N == 0 || (C && bits && scratch), "actnn_bits: null pointer");
  CB_REQUIRE(scratch_bytes >= cogdl_b200_actnn_bits_scratch_bytes(N), "actnn_bits: scratch too small");
  note_kernel("actnn_bits");
  if (N == 0) return COGDL_B200_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int b0 = initial_bits;
  const int64_t n_keys = (int64_t)(b0 - 1) * N;
  int64_t K = (int64_t)b0 * N - target;   // decrements the greedy makes (each lowers sum(b) by 1)
  if (K < 0) K = 0;
  if (K > n_keys) K = n_keys;
  char *w = static_cast<char *>(scratch);
  int *bad = reinterpret_cast<int *>(w);
  uint64_t *keys = reinterpret_cast<uint64_t *>(w + 256);
  uint64_t *sorted = reinterpret_cast<uint64_t *>(w + 256 + align256(7 * N * 8));
  void *temp = w + 256 + 2 * align256(7 * N * 8);
  size_t temp_bytes = sort_temp_bytes(7 * N);
  CB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
  if (n_keys > 0) {
    actnn_alloc_keys_kernel<<<(unsigned)ceil_div(n_keys, kThreads), kThreads, 0, s>>>(C, N, b0, keys, bad);
    CB_LAUNCH_CHECK();
  }
  // C itself never leaves the device: the host reads one status word, so a NaN, infinite or negative C is an error
  int h_bad = 0;
  CB_CUDA(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, s));
  CB_CUDA(cudaStreamSynchronize(s));
  CB_REQUIRE(!h_bad, "actnn_bits: C must be finite and >= 0");
  if (K > 0) {
    CB_CUDA(cub::DeviceRadixSort::SortKeysDescending(temp, temp_bytes, keys, sorted, (int)n_keys, 0, 64, s));
    count_launch();
  }
  actnn_alloc_count_kernel<<<(unsigned)ceil_div(N, kThreads), kThreads, 0, s>>>(C, N, b0, K, sorted, bits);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

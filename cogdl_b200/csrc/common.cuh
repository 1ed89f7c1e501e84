// common.cuh -- shared device/host helpers for libcogdl_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cogdl_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libcogdl_b200 is written for sm_90a (H100) only"
#endif

namespace cogdl_b200 {

// ------------------------------------------------------------------ host side
// SMs of an H100 SXM: caps the grids of the grid-stride kernels at a few waves.
constexpr int NUM_SMS = 132;
int set_error(int code, const char *fmt, ...);
void count_launch(int n = 1);
// Records which kernel instantiation the last dispatching entry point on this thread chose
// (cogdl_b200_last_kernel(); bench.py checks it against the profiled kernel's name).
void note_kernel(const char *fmt, ...);
void append_kernel_note(const char *fmt, ...);   // launch-shape suffix after the instantiation name

#define CB_REQUIRE(cond, ...)                                             \
  do {                                                                    \
    if (!(cond)) return ::cogdl_b200::set_error(COGDL_B200_EINVAL, __VA_ARGS__); \
  } while (0)

#define CB_CUDA(expr)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return ::cogdl_b200::set_error(_e == cudaErrorNoKernelImageForDevice ? COGDL_B200_EDEVICE \
                                                                           : COGDL_B200_ECUDA, \
                                     "%s: %s", #expr, cudaGetErrorString(_e));              \
  } while (0)

// Every launch goes through this: counts it and turns a launch failure into a status code.
#define CB_LAUNCH_CHECK()                  \
  do {                                     \
    ::cogdl_b200::count_launch();          \
    CB_CUDA(cudaPeekAtLastError());        \
  } while (0)

// cudaFuncSetAttribute is per device: a once-flag per (kernel, device), device < 64.  Racing first calls from two
// host threads set the attribute twice, which is harmless.  Returns the current device in *dev.
static inline bool first_use_on_device(unsigned long long &mask, int *dev) {
  *dev = 0;
  if (cudaGetDevice(dev) != cudaSuccess || *dev < 0 || *dev >= 64) return true;
  const unsigned long long bit = 1ull << *dev;
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Plain-old-data view of the hub plan handed to kernels.
struct HubView {
  int chunk_edges;       // 0 => no plan: rows are never skipped / split
  int n_chunks;
  const int2 *chunks;    // (row, first_slot)
  int *counters;
  void *partials;
  int n_segs;            // 0 => no row-stream segments
  const int2 *segs;      // (row_begin, row_end), hub-free
  const int *edge_row;
  int n_empty_rows;
};

static inline HubView hub_view(const cogdl_b200_hub_plan_t *plan) {
  HubView h{0, 0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, 0};
  if (plan && plan->chunk_edges > 0) {
    h.chunk_edges = plan->chunk_edges;
    h.n_chunks = plan->n_chunks;
    h.chunks = reinterpret_cast<const int2 *>(plan->chunks);
    h.counters = plan->counters;
    h.partials = plan->partials;
    if (plan->segs && plan->edge_row && plan->n_segs > 0) {
      h.n_segs = plan->n_segs;
      h.segs = reinterpret_cast<const int2 *>(plan->segs);
      h.edge_row = plan->edge_row;
      h.n_empty_rows = plan->n_empty_rows;
    }
  }
  return h;
}

int check_plan(const cogdl_b200_hub_plan_t *plan, int64_t need_partial_bytes);

// Launch helper of the gather kernels that give GROUP lanes to each of `items` work items (256 threads per block):
// rejects grids beyond int32 under the caller's name `who`, records the instantiation for cogdl_b200_last_kernel()
// (printf-style `fmt`) and launches.
template <typename P, typename... Args>
static int launch_items(void (*kernel)(P), const P &p, int64_t items, int group, cudaStream_t stream, const char *who,
                        const char *fmt, Args... args) {
  const int64_t blocks = ceil_div(items * group, 256);
  if (blocks == 0) return COGDL_B200_OK;
  if (blocks > 0x7fffffffLL)
    return set_error(COGDL_B200_EINVAL, "%s: problem too large for one launch (blocks=%lld)", who, (long long)blocks);
  note_kernel(fmt, args...);
  kernel<<<(unsigned)blocks, 256, 0, stream>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

// ------------------------------------------------------------------ device side
#ifdef __CUDACC__

constexpr unsigned FULL = 0xffffffffu;

// ReLU as torch.relu gives it: a NaN passes through (fmaxf(NaN, 0) would return 0 and hide a diverged value).
__device__ __forceinline__ float relu_nan(float v) { return v < 0.f ? 0.f : v; }

// Streaming (read-once) index/value loads: keep them out of L1 so the gathered feature rows
// own it.  ld.global.nc.L1::no_allocate.
__device__ __forceinline__ int ld_stream(const int *p) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_stream(const float *p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
// Gathered feature rows: read-only path, default caching (hub columns do get reused).
__device__ __forceinline__ float4 ld_gather(const float4 *p) { return __ldg(p); }
__device__ __forceinline__ float2 ld_gather(const float2 *p) { return __ldg(p); }
__device__ __forceinline__ float ld_gather(const float *p) { return __ldg(p); }

// Output rows are written once and never re-read by the kernel: streaming store.
__device__ __forceinline__ void st_stream(float4 *p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream(float2 *p, float2 v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream(float *p, float v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream(int *p, int v) { __stcs(p, v); }

// L2-coherent accesses for inter-CTA partial results (L1 is not coherent across SMs).
__device__ __forceinline__ float4 ld_cg(const float4 *p) { return __ldcg(p); }
__device__ __forceinline__ float2 ld_cg(const float2 *p) { return __ldcg(p); }
__device__ __forceinline__ float ld_cg(const float *p) { return __ldcg(p); }
__device__ __forceinline__ int ld_cg(const int *p) { return __ldcg(p); }
__device__ __forceinline__ void st_cg(float4 *p, float4 v) { __stcg(p, v); }
__device__ __forceinline__ void st_cg(float2 *p, float2 v) { __stcg(p, v); }
__device__ __forceinline__ void st_cg(float *p, float v) { __stcg(p, v); }
__device__ __forceinline__ void st_cg(int *p, int v) { __stcg(p, v); }

// acc += v*x with a separate multiply and add (no FMA contraction): this is what makes the
// SpMM bit-identical to the reference CPU loop `out[ik+t] += val * dense[j+t]`
// (cogdl/operators/spmm/spmm_cpu.cpp:31-33, built without -O => no contraction).
__device__ __forceinline__ float mul_add_rn(float acc, float v, float x) {
  return __fadd_rn(acc, __fmul_rn(v, x));
}
// in-place forms, one per vector type
__device__ __forceinline__ void axpy_rn(float &acc, float v, const float &x) { acc = mul_add_rn(acc, v, x); }
__device__ __forceinline__ void axpy_rn(float2 &acc, float v, const float2 &x) {
  acc.x = mul_add_rn(acc.x, v, x.x);
  acc.y = mul_add_rn(acc.y, v, x.y);
}
__device__ __forceinline__ void axpy_rn(float4 &acc, float v, const float4 &x) {
  acc.x = mul_add_rn(acc.x, v, x.x);
  acc.y = mul_add_rn(acc.y, v, x.y);
  acc.z = mul_add_rn(acc.z, v, x.z);
  acc.w = mul_add_rn(acc.w, v, x.w);
}
__device__ __forceinline__ void add_rn(float &acc, const float &x) { acc = __fadd_rn(acc, x); }
__device__ __forceinline__ void add_rn(float2 &acc, const float2 &x) {
  acc.x = __fadd_rn(acc.x, x.x);
  acc.y = __fadd_rn(acc.y, x.y);
}
__device__ __forceinline__ void add_rn(float4 &acc, const float4 &x) {
  acc.x = __fadd_rn(acc.x, x.x);
  acc.y = __fadd_rn(acc.y, x.y);
  acc.z = __fadd_rn(acc.z, x.z);
  acc.w = __fadd_rn(acc.w, x.w);
}
// elementwise a * b and a - b, correctly rounded (the composition operators of the CompGCN aggregation)
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float2 mul_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float4 mul_rn(float4 a, float4 b) {
  return make_float4(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y), __fmul_rn(a.z, b.z), __fmul_rn(a.w, b.w));
}
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float2 sub_rn(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float4 sub_rn(float4 a, float4 b) {
  return make_float4(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z), __fsub_rn(a.w, b.w));
}
// Attention that carries a dropout mask in its sign bit (GAT attention dropout, edge_softmax.cu MODE 2): a dropped
// entry reads as 0, a kept one as a * scale.  The BIT is tested, not a < 0: a dropped softmax that underflowed to 0
// is stored as -0.0.  A dropped entry is |a| * 0, not a selected 0, so a dropped NaN stays NaN (torch's a * mask * scale).
__device__ __forceinline__ float drop_att(float a, float scale) {
  return __fmul_rn(fabsf(a), __int_as_float(~(__float_as_int(a) >> 31) & __float_as_int(scale)));
}
template <typename VecT> __device__ __forceinline__ VecT vzero();
template <> __device__ __forceinline__ float4 vzero<float4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <> __device__ __forceinline__ float2 vzero<float2>() { return make_float2(0.f, 0.f); }
template <> __device__ __forceinline__ float vzero<float>() { return 0.f; }

template <int WIDTH>
__device__ __forceinline__ int group_max(int v) {
#pragma unroll
  for (int s = WIDTH / 2; s > 0; s >>= 1) v = max(v, __shfl_xor_sync(FULL, v, s));
  return v;
}
__device__ __forceinline__ int warp_max(int v) { return group_max<32>(v); }

// What a group of lanes works on: either one whole row, or one fixed-size edge chunk of a hub
// row.  Items [0, n_chunks) are hub chunks (scheduled first: longest work first), items
// [n_chunks, n_chunks + n_rows) are rows; hub rows are skipped in the row range.
struct WorkItem {
  int row;        // destination row
  int lb, hb;     // edge range
  int slot;       // chunk slot (valid if is_chunk)
  int first;      // first slot of this row's chunks
  int n_row_chunks;
  bool active;
  bool is_chunk;
};

__device__ __forceinline__ WorkItem decode_item(int64_t item, int64_t n_rows, const int *__restrict__ rowptr,
                                                const HubView &hub) {
  WorkItem w;
  w.row = 0; w.lb = 0; w.hb = 0; w.slot = 0; w.first = 0; w.n_row_chunks = 0;
  w.active = false; w.is_chunk = false;
  if (item < hub.n_chunks) {
    const int2 c = __ldg(hub.chunks + item);
    const int rb = __ldg(rowptr + c.x), re = __ldg(rowptr + c.x + 1);
    w.row = c.x;
    w.first = c.y;
    w.slot = (int)item;
    w.lb = rb + ((int)item - c.y) * hub.chunk_edges;
    w.hb = min(w.lb + hub.chunk_edges, re);
    w.n_row_chunks = (re - rb + hub.chunk_edges - 1) / hub.chunk_edges;
    w.active = true;
    w.is_chunk = true;
  } else if (item - hub.n_chunks < n_rows) {
    w.row = (int)(item - hub.n_chunks);
    w.lb = __ldg(rowptr + w.row);
    w.hb = __ldg(rowptr + w.row + 1);
    w.active = !(hub.chunk_edges > 0 && (w.hb - w.lb) > hub.chunk_edges);
    if (!w.active) w.hb = w.lb;
  }
  return w;
}

// Arrival protocol for the chunks of one hub row: every lane has stored its part of the
// partial (st.cg); returns true in all lanes of the group that arrived last.
template <int GROUP>
__device__ __forceinline__ bool hub_arrive_last(const WorkItem &w, const HubView &hub, int gl) {
  __threadfence();   // my partial is visible device-wide before the counter moves
  __syncwarp();
  int old = 0;
  if (w.is_chunk && gl == 0) old = atomicAdd(hub.counters + w.first, 1);
  old = __shfl_sync(FULL, old, 0, GROUP);
  const bool last = w.is_chunk && (old == w.n_row_chunks - 1);
  if (last) {
    if (gl == 0) hub.counters[w.first] = 0;   // leave the counter ready for the next call
    __threadfence();                          // acquire side: partials read after this point
  }
  return last;
}

// The last chunk's combine: folds the n partials of one hub row strictly in chunk order, DEPTH loads in flight, and
// returns the result.  The fold starts from partial 0, not from an identity: 0.0f + -0.0f would turn a -0.0f sum
// into +0.0f.  The row-stream SpMM keeps 8 partials in flight (a 22 K-edge hub has 354: that loop is the kernel's
// tail); the row kernels and scatter_max fold one at a time -- an 8-deep fold there changed their register
// allocation and measured slower (DESIGN 3.2).
template <int DEPTH, typename Load, typename Fold>
__device__ __forceinline__ auto merge_chunks(const int n, Load load, Fold fold) {
  auto s = load(0);
  int q = 1;
  if constexpr (DEPTH > 1) {
    for (; q + DEPTH <= n; q += DEPTH) {
      decltype(s) t[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; ++u) t[u] = load(q + u);
#pragma unroll
      for (int u = 0; u < DEPTH; ++u) fold(s, t[u]);
    }
  }
  for (; q < n; ++q) fold(s, load(q));
  return s;
}

#endif  // __CUDACC__

}  // namespace cogdl_b200

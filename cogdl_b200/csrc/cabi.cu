// cabi.cu -- C-ABI plumbing of libcogdl_b200: error text, device check, launch counter and the
// hub plan (which rows are cut into edge chunks).  See include/cogdl_b200.h.
#include "common.cuh"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstddef>
#include <cstring>

namespace cogdl_b200 {

static thread_local char g_err[512] = {0};
static std::atomic<int64_t> g_launches{0};

int set_error(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static thread_local char g_kernel[256] = {0};
void note_kernel(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_kernel, sizeof(g_kernel), fmt, ap);
  va_end(ap);
}

void append_kernel_note(const char *fmt, ...) {
  const size_t n = strlen(g_kernel);
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_kernel + n, sizeof(g_kernel) - n, fmt, ap);
  va_end(ap);
}

int check_plan(const cogdl_b200_hub_plan_t *plan, int64_t need_partial_bytes) {
  if (!plan || plan->chunk_edges <= 0) return COGDL_B200_OK;
  if (plan->n_chunks < 0 || plan->n_hub_rows < 0)
    return set_error(COGDL_B200_EINVAL, "hub plan: negative counts");
  if (plan->n_chunks == 0) return COGDL_B200_OK;
  if (!plan->chunks || !plan->counters || !plan->hub_rows)
    return set_error(COGDL_B200_EINVAL, "hub plan: null chunk/counter/hub_rows array with n_chunks=%d", plan->n_chunks);
  if (need_partial_bytes > 0 && (!plan->partials || plan->partials_bytes < need_partial_bytes))
    return set_error(COGDL_B200_ESCRATCH, "hub plan: partials scratch too small (have %lld bytes, need %lld)",
                     (long long)plan->partials_bytes, (long long)need_partial_bytes);
  return COGDL_B200_OK;
}

// A row starts a segment iff it is not a hub and (it is row 0, or the previous row is a hub, or the
// cumulative cost P(r) = rowptr[r] + r crosses a multiple of Q between r-1 and r).
__device__ __forceinline__ bool seg_start(const int *rowptr, int64_t r, int T, int Q) {
  const int b = rowptr[r], e = rowptr[r + 1];
  if (e - b > T) return false;
  if (r == 0) return true;
  const int pb = rowptr[r - 1];
  if (b - pb > T) return true;
  return ((int64_t)b + r) / Q != ((int64_t)pb + r - 1) / Q;
}

// counts[0] += #hub rows, [1] += #chunks, [2] += #empty rows, [3] += #segments
__global__ void hub_count_kernel(const int *__restrict__ rowptr, int64_t n_rows, int T, int Q, int *counts) {
  int hubs = 0, chunks = 0, empties = 0, segs = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows;
       r += (int64_t)gridDim.x * blockDim.x) {
    const int deg = rowptr[r + 1] - rowptr[r];
    if (deg > T) {
      hubs += 1;
      chunks += (deg + T - 1) / T;
    }
    if (deg == 0) empties += 1;
    if (Q > 0 && seg_start(rowptr, r, T, Q)) segs += 1;
  }
  for (int s = 16; s > 0; s >>= 1) {
    hubs += __shfl_xor_sync(FULL, hubs, s);
    chunks += __shfl_xor_sync(FULL, chunks, s);
    empties += __shfl_xor_sync(FULL, empties, s);
    segs += __shfl_xor_sync(FULL, segs, s);
  }
  if ((threadIdx.x & 31) == 0) {
    if (hubs) { atomicAdd(counts + 0, hubs); atomicAdd(counts + 1, chunks); }
    if (empties) atomicAdd(counts + 2, empties);
    if (segs) atomicAdd(counts + 3, segs);
  }
}

__global__ void hub_fill_kernel(const int *__restrict__ rowptr, int64_t n_rows, int T, int Q, int *counts,
                                int *hub_rows, int2 *chunks, int2 *segs) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows;
       r += (int64_t)gridDim.x * blockDim.x) {
    const int deg = rowptr[r + 1] - rowptr[r];
    if (deg > T) {
      const int n = (deg + T - 1) / T;
      const int h = atomicAdd(counts + 0, 1);
      const int first = atomicAdd(counts + 1, n);
      hub_rows[h] = (int)r;
      for (int j = 0; j < n; ++j) chunks[first + j] = make_int2((int)r, first);
    }
    if (Q > 0 && segs && seg_start(rowptr, r, T, Q)) {
      int64_t end = r + 1;   // extend to the next hub row / segment start (at most Q rows away)
      while (end < n_rows && (rowptr[end + 1] - rowptr[end]) <= T &&
             ((int64_t)rowptr[end] + end) / Q == ((int64_t)rowptr[end - 1] + end - 1) / Q)
        ++end;
      const int k = atomicAdd(counts + 3, 1);
      segs[k] = make_int2((int)r, (int)end);
    }
  }
}

// edge_row[p] = largest r with rowptr[r] <= p
__global__ void edge_rows_kernel(const int *__restrict__ rowptr, int64_t n_rows, int64_t nnz, int *edge_row) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += stride) {
    int64_t lo = 0, hi = n_rows;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (__ldg(rowptr + mid) <= p) lo = mid; else hi = mid - 1;
    }
    edge_row[p] = (int)lo;
  }
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int cogdl_b200_abi_version(void) { return COGDL_B200_ABI_VERSION; }

extern "C" const char *cogdl_b200_last_error(void) { return g_err; }

extern "C" int64_t cogdl_b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

extern "C" const char *cogdl_b200_last_kernel(void) { return g_kernel; }

extern "C" int cogdl_b200_hub_plan_layout(int64_t *out, int n) {
  typedef cogdl_b200_hub_plan_t P;
  const int64_t v[] = {(int64_t)sizeof(P), offsetof(P, chunk_edges), offsetof(P, n_hub_rows), offsetof(P, n_chunks),
                       offsetof(P, n_empty_rows), offsetof(P, hub_rows), offsetof(P, chunks), offsetof(P, counters),
                       offsetof(P, partials), offsetof(P, partials_bytes), offsetof(P, seg_cost), offsetof(P, n_segs),
                       offsetof(P, segs), offsetof(P, edge_row), offsetof(P, hub_degrees_host)};
  const int m = (int)(sizeof(v) / sizeof(v[0]));
  int k = 0;
  for (; out && k < m && k < n; ++k) out[k] = v[k];
  return k;
}

extern "C" int cogdl_b200_check_device(void) {
  int dev = 0;
  CB_CUDA(cudaGetDevice(&dev));
  int major = 0;
  CB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  if (major != 9)
    return set_error(COGDL_B200_EDEVICE, "device %d has compute capability %d.x; libcogdl_b200 is built for sm_90a only", dev, major);
  return COGDL_B200_OK;
}

static int plan_grid(int64_t n_rows) {
  int64_t b = ceil_div(n_rows, 256);
  if (b > NUM_SMS * 16) b = NUM_SMS * 16;
  if (b < 1) b = 1;
  return (int)b;
}

extern "C" int cogdl_b200_hub_plan_count(const int32_t *rowptr, int64_t n_rows, int32_t chunk_edges,
                                         int32_t seg_cost, int32_t *counts_dev, cogdl_b200_stream_t stream) {
  CB_REQUIRE(rowptr && counts_dev, "cogdl_b200_hub_plan_count: null pointer");
  CB_REQUIRE(n_rows >= 0 && chunk_edges > 0, "cogdl_b200_hub_plan_count: bad size");
  cudaStream_t s = (cudaStream_t)stream;
  CB_CUDA(cudaMemsetAsync(counts_dev, 0, 4 * sizeof(int32_t), s));
  if (n_rows == 0) return COGDL_B200_OK;
  hub_count_kernel<<<plan_grid(n_rows), 256, 0, s>>>(rowptr, n_rows, chunk_edges, seg_cost, counts_dev);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_hub_plan_fill(const int32_t *rowptr, int64_t n_rows, int32_t chunk_edges,
                                        int32_t seg_cost, int32_t *counts_dev, int32_t *hub_rows,
                                        int32_t *chunks, int32_t *segs, cogdl_b200_stream_t stream) {
  CB_REQUIRE(rowptr && counts_dev && hub_rows && chunks, "cogdl_b200_hub_plan_fill: null pointer");
  CB_REQUIRE(n_rows >= 0 && chunk_edges > 0, "cogdl_b200_hub_plan_fill: bad size");
  CB_REQUIRE(seg_cost <= 0 || segs, "cogdl_b200_hub_plan_fill: segs is null but seg_cost > 0");
  cudaStream_t s = (cudaStream_t)stream;
  CB_CUDA(cudaMemsetAsync(counts_dev, 0, 4 * sizeof(int32_t), s));
  if (n_rows == 0) return COGDL_B200_OK;
  hub_fill_kernel<<<plan_grid(n_rows), 256, 0, s>>>(rowptr, n_rows, chunk_edges, seg_cost, counts_dev, hub_rows,
                                                    reinterpret_cast<int2 *>(chunks), reinterpret_cast<int2 *>(segs));
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_edge_rows(const int32_t *rowptr, int64_t n_rows, int64_t nnz, int32_t *edge_row,
                                    cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && nnz >= 0, "cogdl_b200_edge_rows: negative size");
  if (nnz == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && edge_row, "cogdl_b200_edge_rows: null pointer");
  int64_t blocks = ceil_div(nnz, 256);
  if (blocks > NUM_SMS * 32) blocks = NUM_SMS * 32;
  edge_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(rowptr, n_rows, nnz, edge_row);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

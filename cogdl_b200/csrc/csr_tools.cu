// csr_tools.cu -- integer-only structure conversions on the device (sm_90a):
//   csr2csc (+ permutation), row gather by permutation, COO -> CSR index, int64 -> int32.
//
// Replaces: spmm.csr2csc / mhtranspose.csr2csc (cuSPARSE cusparseCsr2cscEx2 with a fresh handle
// and cudaMalloc per call, cogdl/operators/spmm/spmm_kernel.cu:514-532,596-613; mhTranspose.cu:
// 51-111), mhtranspose (mhTranspose.cu:6-49), sampler.coo2csr_cpu_index (single-thread CPU
// counting sort, cogdl/operators/sample/sample.cpp:234-270) and the per-call `.int()` casts
// (cogdl/utils/spmm_utils.py:106).
//
// The stable sort underneath is cub::DeviceRadixSort (header-only template code from the CUDA
// toolkit, compiled into this library -- not a cuSPARSE/torch-sparse dispatch).  These run once
// per graph structure (results are cached by the Python layer), never in the per-step hot loop.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>

namespace cogdl_b200 {

static inline int64_t align256(int64_t x) { return (x + 255) & ~(int64_t)255; }

static int bits_for(int64_t n) {  // bits needed to represent values in [0, n)
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < n) ++b;
  return b;
}

template <typename T>
__global__ void iota_kernel(T *out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (T)i;
}

// ptr[k] = number of sorted keys < k, for k in [0, n_keys]   (lower_bound per bucket)
template <typename KeyT, typename PtrT>
__global__ void bucket_ptr_kernel(const KeyT *__restrict__ sorted, int64_t nnz, int64_t n_buckets, PtrT *ptr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= n_buckets; k += stride) {
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)sorted[mid] < k) lo = mid + 1; else hi = mid;
    }
    ptr[k] = (PtrT)lo;
  }
}

// rowind[q] = row owning CSR position perm[q]   (upper_bound over rowptr)
__global__ void row_of_edge_kernel(const int *__restrict__ rowptr, int64_t n_rows, const int *__restrict__ perm,
                                   int64_t nnz, int *rowind) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nnz; q += stride) {
    const int e = perm[q];
    int64_t lo = 0, hi = n_rows;  // largest r with rowptr[r] <= e
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (__ldg(rowptr + mid) <= e) lo = mid; else hi = mid - 1;
    }
    rowind[q] = (int)lo;
  }
}

__global__ void gather_rows_kernel(const int *__restrict__ perm, const float *__restrict__ in, float *out,
                                   int64_t total, int H) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int64_t q = t / H;
    const int h = (int)(t - q * H);
    out[t] = __ldg(in + (int64_t)__ldg(perm + q) * H + h);
  }
}

__global__ void narrow_kernel(const int64_t *__restrict__ in, int *out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (int)in[i];
}

// Column sums of an edge-aligned [nnz, H] tensor through the transpose (colptr, perm): one thread per
// (item, head), sequential over the item's entries => deterministic.  Hub columns are cut into the
// plan's chunks (pass 1: partial per chunk slot; pass 2: the thread of the row's FIRST slot adds the
// partials in chunk order).  Adjacent threads are adjacent heads of one edge row: 4*H contiguous bytes.
struct ColsumParams {
  const int *colptr;
  const int *perm;
  const float *e;
  float *out;
  int64_t n_cols;
  int H;
  HubView hub;
  float *part;
};

__global__ void colsum_chunk_kernel(const ColsumParams p) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t item = tid / p.H;
  const int h = (int)(tid - item * p.H);
  if (item >= p.hub.n_chunks) return;
  const int2 c = __ldg(p.hub.chunks + item);
  const int cb = __ldg(p.colptr + c.x) + ((int)item - c.y) * p.hub.chunk_edges;
  const int ce = min(cb + p.hub.chunk_edges, __ldg(p.colptr + c.x + 1));
  float acc = 0.f;
  for (int q = cb; q < ce; ++q) acc += __ldg(p.e + (int64_t)__ldg(p.perm + q) * p.H + h);
  p.part[item * p.H + h] = acc;
}

__global__ void colsum_kernel(const ColsumParams p) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t item = tid / p.H;
  const int h = (int)(tid - item * p.H);
  if (item < p.hub.n_chunks) {
    const int2 c = __ldg(p.hub.chunks + item);
    if (c.y != (int)item) return;             // only the first slot of a hub column writes
    const int deg = __ldg(p.colptr + c.x + 1) - __ldg(p.colptr + c.x);
    const int n = (deg + p.hub.chunk_edges - 1) / p.hub.chunk_edges;
    float acc = 0.f;
    for (int q = 0; q < n; ++q) acc += p.part[(item + q) * p.H + h];
    p.out[(int64_t)c.x * p.H + h] = acc;
    return;
  }
  const int64_t col = item - p.hub.n_chunks;
  if (col >= p.n_cols) return;
  const int cb = __ldg(p.colptr + col), ce = __ldg(p.colptr + col + 1);
  if (p.hub.chunk_edges > 0 && ce - cb > p.hub.chunk_edges) return;   // hub column: handled above
  float acc = 0.f;
  for (int q = cb; q < ce; ++q) acc += __ldg(p.e + (int64_t)__ldg(p.perm + q) * p.H + h);
  p.out[col * p.H + h] = acc;
}

static unsigned grid_for(int64_t n) {
  int64_t b = ceil_div(n, 256);
  if (b > NUM_SMS * 32) b = NUM_SMS * 32;
  if (b < 1) b = 1;
  return (unsigned)b;
}

template <typename KeyT>
static int64_t sort_temp_bytes(int64_t nnz) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs<KeyT, KeyT, int64_t>(nullptr, bytes, nullptr, nullptr, nullptr, nullptr, nnz, 0,
                                                       (int)sizeof(KeyT) * 8, 0);
  return (int64_t)bytes;
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_csr2csc_workspace_bytes(int64_t nnz, int64_t n_cols) {
  (void)n_cols;
  if (nnz < 0) return -1;
  return 2 * align256(nnz * 4) + align256(sort_temp_bytes<int>(nnz)) + 256;
}

extern "C" int cogdl_b200_csr2csc(const int32_t *rowptr, const int32_t *colind, int64_t n_rows, int64_t n_cols,
                                  int64_t nnz, int32_t *colptr, int32_t *rowind, int32_t *perm, void *workspace,
                                  int64_t workspace_bytes, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && n_cols >= 0 && nnz >= 0, "cogdl_b200_csr2csc: negative size");
  CB_REQUIRE(rowptr && colptr, "cogdl_b200_csr2csc: null pointer");
  CB_REQUIRE(nnz < 0x7fffffffLL && n_rows < 0x7fffffffLL && n_cols < 0x7fffffffLL,
             "cogdl_b200_csr2csc: sizes must fit int32");
  cudaStream_t s = (cudaStream_t)stream;
  if (nnz == 0) {
    CB_CUDA(cudaMemsetAsync(colptr, 0, (size_t)(n_cols + 1) * sizeof(int32_t), s));
    return COGDL_B200_OK;
  }
  CB_REQUIRE(colind && rowind && perm && workspace, "cogdl_b200_csr2csc: null pointer");
  CB_REQUIRE(workspace_bytes >= cogdl_b200_csr2csc_workspace_bytes(nnz, n_cols),
             "cogdl_b200_csr2csc: workspace too small");
  char *ws = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  int *keys_out = reinterpret_cast<int *>(ws);
  int *vals_in = reinterpret_cast<int *>(ws + align256(nnz * 4));
  void *temp = ws + 2 * align256(nnz * 4);
  size_t temp_bytes = (size_t)sort_temp_bytes<int>(nnz);
  iota_kernel<int><<<grid_for(nnz), 256, 0, s>>>(vals_in, nnz);
  CB_LAUNCH_CHECK();
  // stable LSD radix sort of (column, csr position): CSC order, ascending row inside a column
  CB_CUDA((cub::DeviceRadixSort::SortPairs<int, int, int64_t>(temp, temp_bytes, colind, keys_out, vals_in, perm,
                                                               nnz, 0, bits_for(n_cols), s)));
  count_launch(4);
  bucket_ptr_kernel<int, int><<<grid_for(n_cols + 1), 256, 0, s>>>(keys_out, nnz, n_cols, colptr);
  CB_LAUNCH_CHECK();
  row_of_edge_kernel<<<grid_for(nnz), 256, 0, s>>>(rowptr, n_rows, perm, nnz, rowind);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_gather_rows_f32(const int32_t *perm, const float *in, float *out, int64_t nnz,
                                          int64_t H, cogdl_b200_stream_t stream) {
  CB_REQUIRE(nnz >= 0 && H >= 0, "cogdl_b200_gather_rows_f32: negative size");
  if (nnz == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(perm && in && out, "cogdl_b200_gather_rows_f32: null pointer");
  CB_REQUIRE(H < 0x7fffffffLL, "cogdl_b200_gather_rows_f32: H must fit int32");
  gather_rows_kernel<<<grid_for(nnz * H), 256, 0, (cudaStream_t)stream>>>(perm, in, out, nnz * H, (int)H);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int64_t cogdl_b200_edge_colsum_scratch_bytes(int64_t n_chunks, int64_t H) {
  return n_chunks > 0 && H > 0 ? n_chunks * H * (int64_t)sizeof(float) : 0;
}

extern "C" int cogdl_b200_edge_colsum_f32(const int32_t *colptr, const int32_t *perm, const float *e, float *out,
                                          int64_t n_cols, int64_t H, const cogdl_b200_hub_plan_t *plan,
                                          cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_cols >= 0 && H >= 0, "cogdl_b200_edge_colsum_f32: negative size");
  if (n_cols == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(colptr && perm && e && out, "cogdl_b200_edge_colsum_f32: null pointer");
  CB_REQUIRE(H < 0x7fffffffLL && n_cols < 0x7fffffffLL, "cogdl_b200_edge_colsum_f32: sizes must fit int32");
  ColsumParams p;
  p.colptr = colptr; p.perm = perm; p.e = e; p.out = out; p.n_cols = n_cols; p.H = (int)H;
  p.hub = hub_view(plan);
  p.hub.n_segs = 0;
  int rc = check_plan(plan, cogdl_b200_edge_colsum_scratch_bytes(p.hub.n_chunks, H));
  if (rc) return rc;
  p.part = reinterpret_cast<float *>(p.hub.partials);
  cudaStream_t s = (cudaStream_t)stream;
  if (p.hub.n_chunks > 0) {
    const int64_t b = ceil_div((int64_t)p.hub.n_chunks * H, 256);
    colsum_chunk_kernel<<<(unsigned)b, 256, 0, s>>>(p);
    CB_LAUNCH_CHECK();
  }
  const int64_t blocks = ceil_div(((int64_t)p.hub.n_chunks + n_cols) * H, 256);
  CB_REQUIRE(blocks <= 0x7fffffffLL, "cogdl_b200_edge_colsum_f32: problem too large for one launch");
  colsum_kernel<<<(unsigned)blocks, 256, 0, s>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int64_t cogdl_b200_coo2csr_workspace_bytes(int64_t nnz, int64_t num_nodes) {
  (void)num_nodes;
  if (nnz < 0) return -1;
  return 2 * align256(nnz * 8) + align256(sort_temp_bytes<int64_t>(nnz)) + 256;
}

extern "C" int cogdl_b200_coo2csr_index(const int64_t *row, int64_t nnz, int64_t num_nodes, int64_t *row_ptr,
                                        int64_t *reindex, void *workspace, int64_t workspace_bytes,
                                        cogdl_b200_stream_t stream) {
  CB_REQUIRE(nnz >= 0 && num_nodes >= 0, "cogdl_b200_coo2csr_index: negative size");
  CB_REQUIRE(row_ptr, "cogdl_b200_coo2csr_index: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (nnz == 0) {
    CB_CUDA(cudaMemsetAsync(row_ptr, 0, (size_t)(num_nodes + 1) * sizeof(int64_t), s));
    return COGDL_B200_OK;
  }
  CB_REQUIRE(row && reindex && workspace, "cogdl_b200_coo2csr_index: null pointer");
  CB_REQUIRE(workspace_bytes >= cogdl_b200_coo2csr_workspace_bytes(nnz, num_nodes),
             "cogdl_b200_coo2csr_index: workspace too small");
  char *ws = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  int64_t *keys_out = reinterpret_cast<int64_t *>(ws);
  int64_t *vals_in = reinterpret_cast<int64_t *>(ws + align256(nnz * 8));
  void *temp = ws + 2 * align256(nnz * 8);
  size_t temp_bytes = (size_t)sort_temp_bytes<int64_t>(nnz);
  iota_kernel<int64_t><<<grid_for(nnz), 256, 0, s>>>(vals_in, nnz);
  CB_LAUNCH_CHECK();
  CB_CUDA((cub::DeviceRadixSort::SortPairs<int64_t, int64_t, int64_t>(temp, temp_bytes, row, keys_out, vals_in,
                                                                      reindex, nnz, 0, bits_for(num_nodes), s)));
  count_launch(4);
  bucket_ptr_kernel<int64_t, int64_t><<<grid_for(num_nodes + 1), 256, 0, s>>>(keys_out, nnz, num_nodes, row_ptr);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_narrow_i64_i32(const int64_t *in, int32_t *out, int64_t n, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n >= 0, "cogdl_b200_narrow_i64_i32: negative size");
  if (n == 0) return COGDL_B200_OK;
  CB_REQUIRE(in && out, "cogdl_b200_narrow_i64_i32: null pointer");
  narrow_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(in, out, n);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

// sampler.cu -- neighbour sampling (sample_adj) and induced subgraphs on the device, for sm_90a.
//
// Replaces the reference's single-thread host loops
//   sampler.sample_adj(indptr, indices, node_idx, num_neighbors, replace)   cogdl/operators/sample/sample.cpp:6-146
//   sampler.subgraph(indptr, indices, node_idx)                             cogdl/operators/sample/sample.cpp:148-188
// which Graph.sample_adj / Graph.csr_subgraph call for every mini-batch (cogdl/data/data.py:792-832,
// 850-874; NeighborSampler, cogdl/data/sampler.py:99-104).  int64 in / int64 out, as Graph stores CSR.
//
// What the reference computes, and how the sequential parts are made parallel WITHOUT changing the result:
//   * out_nodes = [batch nodes ..., then every other source node in order of FIRST APPEARANCE in the
//     emitted edge list]; out_indices = position of each edge's source in out_nodes.  The host loop gets
//     this from a running counter.  Here: every non-batch source takes atomicMin(first position q) in a
//     num_nodes-sized scratch (`assoc`), the positions that won are flagged, an exclusive scan of the
//     flags ranks them, id = n_batch + rank.  Same numbering, bit for bit, for ANY edge list.
//   * which edges are emitted: all of a row (num_neighbors < 0), k draws with replacement, or k
//     distinct edges by Robert Floyd's algorithm.  The reference draws with libc rand() (unseeded,
//     sequential, not reproducible); here every draw is a pure function of (seed, batch slot, draw
//     index) -- a counter-based generator (two rounds of the splitmix64 finaliser) that the CPU oracle
//     restates exactly, so a sampled batch is reproducible and checkable bit-for-bit.
//     Deliberate fix (documented divergence): the reference's Floyd loop draws `rand() % j` (0..j-1),
//     which never selects position j except on a collision -- e.g. degree 2, k = 1 ALWAYS returns the
//     first neighbour (sample.cpp:101-104).  We draw from 0..j inclusive (the published algorithm), which
//     gives every k-subset equal probability.  Rows are emitted in Floyd insertion order (the reference's
//     order is std::unordered_set iteration order, i.e. unspecified).
//   * replace = true on a degree-0 row: the reference computes rand() % 0 (SIGFPE); we emit no edge.
// `assoc` scratch contract: int32[num_nodes], every entry COGDL_B200_SAMPLE_UNSEEN (0x7fffffff) on entry;
// restored to that state before the fill call returns, so one allocation serves every batch.
#include "common.cuh"
#include "rng.cuh"

#include <cub/device/device_scan.cuh>

namespace cogdl_b200 {

constexpr int UNSEEN = 0x7fffffff;

__device__ __forceinline__ int64_t row_count(int64_t deg, int64_t k, int replace) {
  if (k < 0) return deg;
  if (replace) return deg > 0 ? k : 0;
  return deg < k ? deg : k;
}

__global__ void sample_count_kernel(const int64_t *__restrict__ indptr, const int64_t *__restrict__ node_idx,
                                    int64_t n_batch, int64_t k, int replace, int64_t *counts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_batch) return;
  const int64_t node = node_idx[i];
  counts[i] = row_count(indptr[node + 1] - indptr[node], k, replace);
}

// One warp per batch row: writes the GLOBAL edge positions of the row's picks to out_edges[o .. o+cnt).
__global__ void __launch_bounds__(256) sample_pick_kernel(const int64_t *__restrict__ indptr,
                                                          const int64_t *__restrict__ node_idx, int64_t n_batch,
                                                          int64_t k, int replace, uint64_t seed,
                                                          const int64_t *__restrict__ out_indptr, int64_t *out_edges) {
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_batch) return;
  const int64_t node = node_idx[i];
  const int64_t rs = indptr[node], deg = indptr[node + 1] - rs;
  const int64_t o = out_indptr[i];
  const int64_t cnt = out_indptr[i + 1] - o;
  if (cnt == 0) return;
  if (k < 0 || (!replace && deg <= k)) {          // the whole row, CSR order
    for (int64_t t = lane; t < cnt; t += 32) out_edges[o + t] = rs + t;
    return;
  }
  if (replace) {
    for (int64_t t = lane; t < cnt; t += 32) out_edges[o + t] = rs + (int64_t)(draw(seed, i, t) % (uint64_t)deg);
    return;
  }
  // Floyd: for j = deg-k .. deg-1: t ~ U{0..j}; take t unless already taken, else take j.
  int64_t have = 0;
  for (int64_t j = deg - k; j < deg; ++j, ++have) {
    const int64_t t = (int64_t)(draw(seed, i, have) % (uint64_t)(j + 1));
    bool hit = false;
    for (int64_t q = lane; q < have; q += 32) hit |= (out_edges[o + q] == rs + t);
    const bool taken = __any_sync(FULL, hit);
    __syncwarp();
    if (lane == 0) out_edges[o + have] = rs + (taken ? j : t);
    __syncwarp();
  }
}

__global__ void mark_batch_kernel(const int64_t *__restrict__ node_idx, int64_t n_batch, int *assoc,
                                  int64_t *out_nodes) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_batch) return;
  assoc[node_idx[i]] = (int)i;
  if (out_nodes) out_nodes[i] = node_idx[i];
}

__global__ void first_touch_kernel(const int64_t *__restrict__ indices, const int64_t *__restrict__ out_edges,
                                   int64_t n_edges, int n_batch, int *assoc) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_edges) return;
  const int64_t s = indices[out_edges[q]];
  if (assoc[s] >= n_batch) atomicMin(assoc + s, n_batch + (int)q);
}

__global__ void flag_first_kernel(const int64_t *__restrict__ indices, const int64_t *__restrict__ out_edges,
                                  int64_t n_edges, int n_batch, const int *__restrict__ assoc, int *flags) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_edges) return;
  flags[q] = (assoc[indices[out_edges[q]]] == n_batch + (int)q) ? 1 : 0;
}

__global__ void relabel_kernel(const int64_t *__restrict__ indices, const int64_t *__restrict__ out_edges,
                               int64_t n_edges, int n_batch, const int *__restrict__ assoc,
                               const int *__restrict__ flags, const int *__restrict__ rank, int64_t *out_indices,
                               int64_t *out_nodes, int64_t *n_out_nodes) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_edges) return;
  const int64_t s = indices[out_edges[q]];
  const int a = assoc[s];
  if (a < n_batch) {
    out_indices[q] = a;
  } else {
    const int p = a - n_batch;                 // position of the first appearance of s
    const int id = n_batch + rank[p];
    out_indices[q] = id;
    if (p == (int)q) out_nodes[id] = s;
  }
  if (q == n_edges - 1) *n_out_nodes = (int64_t)n_batch + rank[q] + flags[q];
}

__global__ void reset_assoc_kernel(const int64_t *__restrict__ indices, const int64_t *__restrict__ out_edges,
                                   int64_t n_edges, const int64_t *__restrict__ node_idx, int64_t n_batch, int *assoc) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_batch) assoc[node_idx[t]] = UNSEEN;
  if (t < n_edges && indices) assoc[indices[out_edges[t]]] = UNSEEN;
}

__global__ void set_scalar_kernel(int64_t *p, int64_t v) { *p = v; }

// ---------------------------------------------------------------- induced subgraph
// One warp per listed node: count / emit the edges whose source is listed too (CSR order kept).
template <bool FILL>
__global__ void __launch_bounds__(256) subgraph_kernel(const int64_t *__restrict__ indptr,
                                                       const int64_t *__restrict__ indices,
                                                       const int64_t *__restrict__ node_idx, int64_t n_sub,
                                                       const int *__restrict__ assoc, int64_t *counts,
                                                       const int64_t *__restrict__ out_indptr, int64_t *out_indices,
                                                       int64_t *out_edges) {
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_sub) return;
  const int64_t node = node_idx[i];
  const int64_t rs = indptr[node], re = indptr[node + 1];
  int64_t base = FILL ? out_indptr[i] : 0;
  for (int64_t e0 = rs; e0 < re; e0 += 32) {
    const int64_t e = e0 + lane;
    int a = UNSEEN;
    if (e < re) a = assoc[indices[e]];
    const bool keep = a != UNSEEN;
    const unsigned m = __ballot_sync(FULL, keep);
    if (FILL && keep) {
      const int64_t dst = base + __popc(m & ((1u << lane) - 1u));
      out_indices[dst] = a;
      out_edges[dst] = e;
    }
    base += __popc(m);
  }
  if (!FILL && lane == 0) counts[i] = base;
}

static inline unsigned blocks_for(int64_t n, int per = 256) { return (unsigned)ceil_div(n > 0 ? n : 1, per); }

}  // namespace cogdl_b200

using namespace cogdl_b200;

static size_t scan_temp_bytes_i64(int64_t n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum((void *)nullptr, b, (const int64_t *)nullptr, (int64_t *)nullptr, (int)(n > 0 ? n : 1));
  return b;
}
static size_t scan_temp_bytes_i32(int64_t n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum((void *)nullptr, b, (const int *)nullptr, (int *)nullptr, (int)(n > 0 ? n : 1));
  return b;
}
static inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

extern "C" int64_t cogdl_b200_sample_workspace_bytes(int64_t n_batch, int64_t n_edges) {
  const int64_t nb = n_batch + 1, ne = n_edges > 0 ? n_edges : 1;
  return (int64_t)(align256((size_t)nb * 8) + align256(scan_temp_bytes_i64(nb)) + 2 * align256((size_t)ne * 4) +
                   align256(scan_temp_bytes_i32(ne)));
}

// Phase 1: out_indptr[0..n_batch] (device) = exclusive scan of the per-row pick counts.  The caller reads
// out_indptr[n_batch] (one 8-byte D2H) to size the outputs of phase 2.
extern "C" int cogdl_b200_sample_adj_count(const int64_t *indptr, const int64_t *node_idx, int64_t n_batch,
                                           int64_t num_neighbors, int32_t replace, int64_t *out_indptr,
                                           void *workspace, int64_t workspace_bytes, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_batch >= 0 && n_batch < 0x7fffffffLL, "cogdl_b200_sample_adj_count: bad batch size");
  CB_REQUIRE(indptr && out_indptr && (node_idx || n_batch == 0), "cogdl_b200_sample_adj_count: null pointer");
  CB_REQUIRE(workspace && workspace_bytes >= cogdl_b200_sample_workspace_bytes(n_batch, 0),
             "cogdl_b200_sample_adj_count: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  char *w = (char *)workspace;
  int64_t *counts = (int64_t *)w;
  w += align256((size_t)(n_batch + 1) * 8);
  size_t tb = scan_temp_bytes_i64(n_batch + 1);
  CB_CUDA(cudaMemsetAsync(counts + n_batch, 0, 8, s));
  if (n_batch > 0) {
    sample_count_kernel<<<blocks_for(n_batch), 256, 0, s>>>(indptr, node_idx, n_batch, num_neighbors, replace, counts);
    CB_LAUNCH_CHECK();
  }
  CB_CUDA(cub::DeviceScan::ExclusiveSum(w, tb, counts, out_indptr, (int)(n_batch + 1), s));
  count_launch();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_sample_adj_fill(const int64_t *indptr, const int64_t *indices, const int64_t *node_idx,
                                          int64_t n_batch, int64_t num_nodes, int64_t num_neighbors, int32_t replace,
                                          uint64_t seed, const int64_t *out_indptr, int64_t n_edges, int32_t *assoc,
                                          int64_t *out_indices, int64_t *out_edges, int64_t *out_nodes,
                                          int64_t *n_out_nodes_dev, void *workspace, int64_t workspace_bytes,
                                          cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_batch >= 0 && n_edges >= 0 && num_nodes >= 0, "cogdl_b200_sample_adj_fill: negative size");
  CB_REQUIRE(n_batch + n_edges < 0x7ffffffeLL, "cogdl_b200_sample_adj_fill: batch + sampled edges must fit int32");
  CB_REQUIRE(indptr && indices && assoc && out_indptr && out_nodes && n_out_nodes_dev && (node_idx || n_batch == 0),
             "cogdl_b200_sample_adj_fill: null pointer");
  CB_REQUIRE(n_edges == 0 || (out_indices && out_edges), "cogdl_b200_sample_adj_fill: null output");
  CB_REQUIRE(workspace && workspace_bytes >= cogdl_b200_sample_workspace_bytes(n_batch, n_edges),
             "cogdl_b200_sample_adj_fill: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  char *w = (char *)workspace;
  w += align256((size_t)(n_batch + 1) * 8) + align256(scan_temp_bytes_i64(n_batch + 1));
  int *flags = (int *)w;
  w += align256((size_t)(n_edges > 0 ? n_edges : 1) * 4);
  int *rank = (int *)w;
  w += align256((size_t)(n_edges > 0 ? n_edges : 1) * 4);
  size_t tb = scan_temp_bytes_i32(n_edges);
  if (n_batch > 0) {
    mark_batch_kernel<<<blocks_for(n_batch), 256, 0, s>>>(node_idx, n_batch, assoc, out_nodes);
    CB_LAUNCH_CHECK();
  }
  if (n_edges == 0) {   // no edge survives: the node list is the batch itself
    set_scalar_kernel<<<1, 1, 0, s>>>(n_out_nodes_dev, n_batch);
    CB_LAUNCH_CHECK();
  } else {
    sample_pick_kernel<<<blocks_for(n_batch * 32), 256, 0, s>>>(indptr, node_idx, n_batch, num_neighbors, replace, seed,
                                                               out_indptr, out_edges);
    CB_LAUNCH_CHECK();
    first_touch_kernel<<<blocks_for(n_edges), 256, 0, s>>>(indices, out_edges, n_edges, (int)n_batch, assoc);
    CB_LAUNCH_CHECK();
    flag_first_kernel<<<blocks_for(n_edges), 256, 0, s>>>(indices, out_edges, n_edges, (int)n_batch, assoc, flags);
    CB_LAUNCH_CHECK();
    CB_CUDA(cub::DeviceScan::ExclusiveSum(w, tb, flags, rank, (int)n_edges, s));
    count_launch();
    relabel_kernel<<<blocks_for(n_edges), 256, 0, s>>>(indices, out_edges, n_edges, (int)n_batch, assoc, flags, rank,
                                                       out_indices, out_nodes, n_out_nodes_dev);
    CB_LAUNCH_CHECK();
  }
  const int64_t m = n_batch > n_edges ? n_batch : n_edges;
  if (m > 0) {
    reset_assoc_kernel<<<blocks_for(m), 256, 0, s>>>(n_edges > 0 ? indices : nullptr, out_edges, n_edges, node_idx, n_batch, assoc);
    CB_LAUNCH_CHECK();
  }
  return COGDL_B200_OK;
}

// Induced subgraph, phase 1: marks assoc (node_idx[i] -> i), counts kept edges per listed node and scans.
// assoc stays marked until cogdl_b200_subgraph_fill (always call it, even when no edge survives).
extern "C" int cogdl_b200_subgraph_count(const int64_t *indptr, const int64_t *indices, const int64_t *node_idx,
                                         int64_t n_sub, int32_t *assoc, int64_t *out_indptr, void *workspace,
                                         int64_t workspace_bytes, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_sub >= 0 && n_sub < 0x7fffffffLL, "cogdl_b200_subgraph_count: bad node count");
  CB_REQUIRE(indptr && indices && assoc && out_indptr && (node_idx || n_sub == 0), "cogdl_b200_subgraph_count: null pointer");
  CB_REQUIRE(workspace && workspace_bytes >= cogdl_b200_sample_workspace_bytes(n_sub, 0),
             "cogdl_b200_subgraph_count: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  char *w = (char *)workspace;
  int64_t *counts = (int64_t *)w;
  w += align256((size_t)(n_sub + 1) * 8);
  size_t tb = scan_temp_bytes_i64(n_sub + 1);
  CB_CUDA(cudaMemsetAsync(counts + n_sub, 0, 8, s));
  if (n_sub > 0) {
    mark_batch_kernel<<<blocks_for(n_sub), 256, 0, s>>>(node_idx, n_sub, assoc, nullptr);
    CB_LAUNCH_CHECK();
    subgraph_kernel<false><<<blocks_for(n_sub * 32), 256, 0, s>>>(indptr, indices, node_idx, n_sub, assoc, counts, nullptr,
                                                                 nullptr, nullptr);
    CB_LAUNCH_CHECK();
  }
  CB_CUDA(cub::DeviceScan::ExclusiveSum(w, tb, counts, out_indptr, (int)(n_sub + 1), s));
  count_launch();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_subgraph_fill(const int64_t *indptr, const int64_t *indices, const int64_t *node_idx,
                                        int64_t n_sub, int32_t *assoc, const int64_t *out_indptr, int64_t *out_indices,
                                        int64_t *out_edges, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_sub >= 0, "cogdl_b200_subgraph_fill: bad node count");
  CB_REQUIRE(indptr && indices && assoc && out_indptr && (node_idx || n_sub == 0), "cogdl_b200_subgraph_fill: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_sub == 0) return COGDL_B200_OK;
  if (out_indices && out_edges) {
    subgraph_kernel<true><<<blocks_for(n_sub * 32), 256, 0, s>>>(indptr, indices, node_idx, n_sub, assoc, nullptr, out_indptr,
                                                                out_indices, out_edges);
    CB_LAUNCH_CHECK();
  }
  reset_assoc_kernel<<<blocks_for(n_sub), 256, 0, s>>>(nullptr, nullptr, 0, node_idx, n_sub, assoc);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" uint64_t cogdl_b200_sample_draw(uint64_t seed, int64_t slot, int64_t k) { return draw(seed, slot, k); }

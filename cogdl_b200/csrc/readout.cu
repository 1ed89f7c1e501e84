// readout.cu -- SortPool's per-graph top-k selection (DGCNN, cogdl/models/nn/sortpool.py:105-126), sm_90a.
//
// For graph g (row g of the membership CSR: its columns are the graph's nodes) the selection names the min(k, n_g)
// nodes with the largest key, in descending key order, ties to the lower node index, NaN above +inf, -0 equal to +0
// (the order of a stable torch.sort(descending=True)).  The reference pads every graph to the largest graph of the
// batch with a fill value, sorts the padding with the data, cuts or pads to k and replaces the fill value by 0: the same
// rows, at the cost of a dense [B, max_n, F] copy and two host reads.
//
// The keys are the bit patterns of the feature matrix's last column and are ordered with integer operations only; the
// kernel reads no other feature.  It writes the selection as a CSR with k rows per graph (row g*k + r holds the r-th
// selected node, or nothing past n_g), so the pooled rows are one SpMM over it and their gradient is the scatter of
// scatter_max's backward: the row movement runs on those entry points.
//
// One block per graph.  A graph of at most k nodes is loaded whole into shared memory.  A larger graph is narrowed
// by a radix select of the k-th largest key over the order-preserving uint32 image of the keys, 8 bits per pass,
// each pass streaming the graph's keys into a shared-memory histogram (integer counts: the result does not depend on
// the order of the atomics); an ordered compaction (block scans in node order) then takes every key above the
// threshold and the first `need` keys equal to it, exactly k survivors.  The survivors are sorted in shared memory
// (bitonic, on a 64-bit composite of the key and the complemented node index, so the order is total).
#include "common.cuh"

namespace cogdl_b200 {
namespace {

constexpr int SP_THREADS = 256;
constexpr int SP_MAX_K = COGDL_B200_SORT_POOL_MAX_K;

// Order-preserving image of an IEEE binary32 bit pattern: a < b  <=>  key(a) < key(b); every NaN (exponent all ones,
// mantissa not 0, either sign) maps above +inf, -0 and +0 to one key.
__device__ __forceinline__ uint32_t sort_key(uint32_t b) {
  const uint32_t mag = b & 0x7fffffffu;
  if (mag > 0x7f800000u) return 0xffffffffu;
  if (mag == 0u) return 0x80000000u;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Larger composite = earlier in the output: key descending, then node ascending.
__device__ __forceinline__ unsigned long long composite(uint32_t key, int node) {
  return ((unsigned long long)key << 32) | (uint32_t)(~(uint32_t)node);
}

__device__ __forceinline__ int composite_node(unsigned long long c) { return (int)(~(uint32_t)c); }

// Exclusive scan of v over the block (SP_THREADS threads); *total gets the block sum.  Ends with a barrier.
__device__ __forceinline__ int block_excl_scan(int v, int *s_warp, int *total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(FULL, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < SP_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(FULL, w, d);
      if (lane >= d) w += o;
    }
    if (lane < SP_THREADS / 32) s_warp[lane] = w;   // inclusive warp prefix
  }
  __syncthreads();
  const int before = (warp > 0 ? s_warp[warp - 1] : 0) + incl - v;
  *total = s_warp[SP_THREADS / 32 - 1];
  __syncthreads();
  return before;
}

struct SortPoolParams {
  const int32_t *rowptr;
  const int32_t *colind;
  const uint32_t *key_bits;   // [n_x_rows]
  const int32_t *sel_off;     // [n_graphs]: selected nodes of the graphs before g
  int32_t *idx;               // [n_graphs, k]
  int32_t *sel_rowptr;        // [n_graphs * k + 1]
  int32_t *sel_colind;        // [>= total selected]
  int64_t n_graphs;
  int k;
};

__global__ void __launch_bounds__(SP_THREADS) sort_pool_select_kernel(SortPoolParams p) {
  __shared__ unsigned long long s_sel[SP_MAX_K];
  __shared__ int s_hist[256];
  __shared__ int s_warp[SP_THREADS / 32];
  __shared__ uint32_t s_prefix;
  __shared__ int s_need;
  const int tid = threadIdx.x;
  const int64_t g = blockIdx.x;
  const int beg = p.rowptr[g];
  const int n = p.rowptr[g + 1] - beg;
  const int k = p.k;
  const int m = n < k ? n : k;
  const uint32_t *keys = p.key_bits;
  const int32_t *nodes = p.colind + beg;

  if (n <= k) {
    for (int i = tid; i < n; i += SP_THREADS) {
      const int node = nodes[i];
      s_sel[i] = composite(sort_key(__ldg(keys + node)), node);
    }
  } else {
    // Radix select: after the pass at `shift`, prefix holds the top bits of the k-th largest key and need the rank
    // of that key among the keys that share those bits.
    uint32_t prefix = 0, mask = 0;
    int need = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += SP_THREADS) s_hist[i] = 0;
      __syncthreads();
      int i = tid;
      for (; i + 3 * SP_THREADS < n; i += 4 * SP_THREADS) {   // four independent loads in flight per thread
        uint32_t kk[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) kk[u] = sort_key(__ldg(keys + nodes[i + u * SP_THREADS]));
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if ((kk[u] & mask) == prefix) atomicAdd(&s_hist[(kk[u] >> shift) & 255u], 1);
      }
      for (; i < n; i += SP_THREADS) {
        const uint32_t key = sort_key(__ldg(keys + nodes[i]));
        if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int above = 0, b = 255;
        for (; b > 0; --b) {
          if (above + s_hist[b] >= need) break;
          above += s_hist[b];
        }
        s_prefix = prefix | ((uint32_t)b << shift);
        s_need = need - above;
      }
      __syncthreads();
      prefix = s_prefix;
      need = s_need;
      mask |= 0xffu << shift;
    }
    // prefix is now the k-th largest key: take every key above it and the first `need` keys equal to it, in node
    // order.  A taken key's slot is (keys above it before it) + min(keys equal to it before it, need).
    int gt_seen = 0, eq_seen = 0;
    for (int c0 = 0; c0 < n; c0 += SP_THREADS) {
      const int i = c0 + tid;
      int node = 0;
      uint32_t key = 0;
      bool gt = false, eq = false;
      if (i < n) {
        node = nodes[i];
        key = sort_key(__ldg(keys + node));
        gt = key > prefix;
        eq = key == prefix;
      }
      int total;
      const int before = block_excl_scan(((int)gt << 16) | (int)eq, s_warp, &total);   // <= 256 of each per chunk
      const int gt_before = gt_seen + (before >> 16), eq_before = eq_seen + (before & 0xffff);
      if (gt || (eq && eq_before < need)) s_sel[gt_before + (eq_before < need ? eq_before : need)] = composite(key, node);
      gt_seen += total >> 16;
      eq_seen += total & 0xffff;
    }
  }
  // Bitonic sort of s_sel[0, m) descending, padded to a power of two with 0 (below every composite: key >= 0x007fffff).
  int P = 1;
  while (P < m) P <<= 1;
  for (int i = m + tid; i < P; i += SP_THREADS) s_sel[i] = 0ull;
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = tid; t < P / 2; t += SP_THREADS) {
        const int i = 2 * t - (t & (stride - 1));
        const int j = i + stride;
        const bool up = (i & size) == 0;
        const unsigned long long a = s_sel[i], b = s_sel[j];
        if ((a < b) == up) {
          s_sel[i] = b;
          s_sel[j] = a;
        }
      }
    }
  }
  __syncthreads();
  const int off = p.sel_off[g];
  int32_t *idx = p.idx + g * k;
  int32_t *rp = p.sel_rowptr + g * k;
  for (int r = tid; r < k; r += SP_THREADS) {
    const int node = r < m ? composite_node(s_sel[r]) : -1;
    idx[r] = node;
    rp[r] = off + (r < m ? r : m);
    if (r < m) p.sel_colind[off + r] = node;
  }
  if (g == p.n_graphs - 1 && tid == 0) p.sel_rowptr[p.n_graphs * k] = off + m;
}

}  // namespace
}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_sort_pool_max_k(void) { return SP_MAX_K; }

extern "C" int cogdl_b200_sort_pool_select(const int32_t *rowptr, const int32_t *colind, const uint32_t *key_bits,
                                           int64_t n_x_rows, int64_t n_graphs, int64_t k, const int32_t *sel_off,
                                           int32_t *idx, int32_t *sel_rowptr, int32_t *sel_colind,
                                           cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_sort_pool_select";
  CB_REQUIRE(n_x_rows >= 0 && n_graphs >= 0, "%s: negative size", who);
  CB_REQUIRE(k >= 1 && k <= SP_MAX_K, "%s: k = %lld is outside [1, %d]", who, (long long)k, SP_MAX_K);
  CB_REQUIRE(n_x_rows < 0x7fffffffLL && n_graphs * k < 0x7fffffffLL, "%s: sizes must fit int32", who);
  cudaStream_t s = (cudaStream_t)stream;
  if (n_graphs == 0) {
    CB_REQUIRE(sel_rowptr, "%s: null pointer", who);
    CB_CUDA(cudaMemsetAsync(sel_rowptr, 0, sizeof(int32_t), s));
    return COGDL_B200_OK;
  }
  CB_REQUIRE(rowptr && colind && sel_off && idx && sel_rowptr && sel_colind && (key_bits || n_x_rows == 0),
             "%s: null pointer", who);
  SortPoolParams p;
  p.rowptr = rowptr; p.colind = colind; p.key_bits = key_bits; p.sel_off = sel_off; p.idx = idx;
  p.sel_rowptr = sel_rowptr; p.sel_colind = sel_colind; p.n_graphs = n_graphs; p.k = (int)k;
  note_kernel("cogdl_b200::sort_pool_select_kernel");
  sort_pool_select_kernel<<<(unsigned)n_graphs, SP_THREADS, 0, s>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

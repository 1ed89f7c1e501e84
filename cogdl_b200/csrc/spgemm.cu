// spgemm.cu -- sparse x sparse product C = A.B (CSR, fp32 values) and its value gradients, sm_90a.
//
// Replaces torch_sparse.spspmm (cuSPARSE SpGEMM), which CogDL's GTN, SRGCN and Graph U-Net import at module
// level (cogdl/models/nn/gtn.py:7, srgcn.py:6, cogdl/utils/srgcn_utils.py:7, graph_unet.py:9).
//
// Two phases, as the sampler's count -> fill:
//   count: the distinct columns of every output row -> rowptrC (int64 totals, one host read to reject nnz > INT32_MAX)
//   fill : the sorted columns of every row, then its values.
// Rows are binned by bound = min(sum_{k in A_i} deg_B(k), n), the most distinct columns the row can have:
//   bound == 0            nothing to do
//   bound <= WARP_CAP     one warp, a shared-memory hash table of 2*WARP_CAP slots, rank sort of the keys
//   bound <= BLOCK_CAP    one block, a shared-memory hash table of 2*BLOCK_CAP slots, cub block radix sort
//   larger                one block with a dense bitmap of the n columns in global scratch (LARGE_SLOTS blocks, each
//                         with its own bitmap and word prefix sums): the column's position in the row is the prefix
//                         popcount, so a row whose output is all of n needs no table at all.
// Values: for a row, A's entries are walked in CSR order; for each k the group's threads take B_k's entries in
// parallel.  B_k's columns are unique, so no two threads touch one output slot within a k, and a barrier separates
// the k's: every output is acc = fmaf(a_ik, b_kj, acc) in (A order, B order), from 0, with no float atomics.  No row
// is split, so every row is bit-identical to the sequential Gustavson loop in that order and results are
// reproducible run to run.
//
// Backward (each output written once, deterministic; one warp per entry, a fixed-shape lane reduction):
//   dA[p=(i,k)] = sum_{q in B_k} b_q dC[i, col_B(q)]
//   dB[q=(k,j)] = sum_{p in column k of A} a_p dC[row(p), j]        (A's transpose from cogdl_b200_csr2csc + perm)
// dC[i, j] is found by binary search in C's sorted row i.
#include "common.cuh"

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

namespace cogdl_b200 {

constexpr int SPG_WARP_CAP = 256;
constexpr int SPG_BLOCK_CAP = 4096;
constexpr int SPG_BLOCK_THREADS = 256;
constexpr int SPG_WARPS = 8;            // warps per block of the warp tier
constexpr int SPG_LARGE_SLOTS = 132;    // concurrent blocks of the bitmap tier (one per SM)

struct SpgParams {
  const int *rpA, *colA;
  const float *valA;
  const int *rpB, *colB;
  const float *valB;
  int m, n, words;
  const int *rpC;
  int *colC;
  float *valC;
  long long *cnt;    // count phase: distinct columns per row
  int *lists;        // [3][m] rows of the warp, block and bitmap tiers
  int *list_n;       // [3]
  unsigned *bits;    // [SPG_LARGE_SLOTS][words], zero between rows
  int *wordpos;      // [SPG_LARGE_SLOTS][words]
};

template <int GROUP>
__device__ __forceinline__ void group_sync() {
  if constexpr (GROUP == 32) __syncwarp(); else __syncthreads();
}

// Fibonacci hashing: the HIGH bits of j * 2^32/phi (the low bits of an odd multiple depend only on j mod TS, so a
// column set with a stride of TS would share one slot)
template <int TS>
__device__ __forceinline__ unsigned spg_hash(int j) {
  static_assert((TS & (TS - 1)) == 0 && TS >= 2, "table size must be a power of two");
  constexpr int BITS = __builtin_ctz(TS);
  return ((unsigned)j * 0x9E3779B1u) >> (32 - BITS);
}

template <int TS>
__device__ __forceinline__ int hash_insert(int *keys, int j) {
  unsigned h = spg_hash<TS>(j);
  while (true) {
    const int prev = atomicCAS(keys + h, -1, j);
    if (prev == -1) return 1;
    if (prev == j) return 0;
    h = (h + 1) & (TS - 1);
  }
}

template <int TS>
__device__ __forceinline__ int hash_find(const int *keys, int j) {
  unsigned h = spg_hash<TS>(j);
  while (keys[h] != j) h = (h + 1) & (TS - 1);
  return (int)h;
}

__global__ void spg_classify_kernel(const SpgParams p, bool count) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < p.m; row += nw) {
    long long ub = 0;
    for (int q = __ldg(p.rpA + row) + lane; q < __ldg(p.rpA + row + 1); q += 32) {
      const int k = __ldg(p.colA + q);
      ub += __ldg(p.rpB + k + 1) - __ldg(p.rpB + k);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) ub += __shfl_xor_sync(FULL, ub, off);
    if (lane == 0) {
      const long long bound = ub < p.n ? ub : p.n;
      const int tier = bound == 0 ? -1 : bound <= SPG_WARP_CAP ? 0 : bound <= SPG_BLOCK_CAP ? 1 : 2;
      if (tier < 0) {
        if (count) p.cnt[row] = 0;
      } else {
        const int at = atomicAdd(p.list_n + tier, 1);
        p.lists[(int64_t)tier * p.m + at] = (int)row;
      }
    }
  }
}

// One row on a hash table of 2*CAP slots, GROUP threads (thread t).  keys/pos: [2*CAP]; acc: [CAP] (also the compacted
// key list); ctr: one int.  Ends with a group barrier, so the caller can move on to its next row.
template <int GROUP, int CAP, bool FILL, typename SortStorage>
__device__ __forceinline__ void hash_row(const SpgParams &p, int row, int t, int *keys, int *pos, float *acc, int *ctr,
                                         SortStorage *sort_tmp) {
  constexpr int TS = 2 * CAP;
  for (int h = t; h < TS; h += GROUP) keys[h] = -1;
  if (t == 0) *ctr = 0;
  group_sync<GROUP>();
  const int ab = __ldg(p.rpA + row), ae = __ldg(p.rpA + row + 1);
  int mine = 0;
  for (int e = ab; e < ae; ++e) {
    const int k = __ldg(p.colA + e);
    for (int q = __ldg(p.rpB + k) + t; q < __ldg(p.rpB + k + 1); q += GROUP) mine += hash_insert<TS>(keys, __ldg(p.colB + q));
  }
  if (mine) atomicAdd(ctr, mine);
  group_sync<GROUP>();
  const int c = *ctr;
  if constexpr (!FILL) {
    if (t == 0) p.cnt[row] = c;
    group_sync<GROUP>();
    return;
  } else {
    int *list = reinterpret_cast<int *>(acc);
    group_sync<GROUP>();
    if (t == 0) *ctr = 0;
    group_sync<GROUP>();
    for (int h = t; h < TS; h += GROUP) {
      const int key = keys[h];
      if (key >= 0) list[atomicAdd(ctr, 1)] = key;
    }
    group_sync<GROUP>();
    const int base = __ldg(p.rpC + row);
    if constexpr (GROUP == 32) {
      // rank sort: the rank of a key is the number of keys below it (c <= CAP keys, c*c/32 compares per lane)
      for (int e = t; e < c; e += GROUP) {
        const int key = list[e];
        int r = 0;
        for (int x = 0; x < c; ++x) r += list[x] < key;
        p.colC[base + r] = key;
        pos[hash_find<TS>(keys, key)] = r;
      }
    } else {
      constexpr int IPT = CAP / GROUP;
      int items[IPT];
#pragma unroll
      for (int u = 0; u < IPT; ++u) items[u] = t * IPT + u < c ? list[t * IPT + u] : 0x7fffffff;
      cub::BlockRadixSort<int, GROUP, IPT>(*sort_tmp).Sort(items);
#pragma unroll
      for (int u = 0; u < IPT; ++u) {
        const int r = t * IPT + u;
        if (r < c) {
          p.colC[base + r] = items[u];
          pos[hash_find<TS>(keys, items[u])] = r;
        }
      }
    }
    group_sync<GROUP>();
    for (int r = t; r < c; r += GROUP) acc[r] = 0.f;
    group_sync<GROUP>();
    for (int e = ab; e < ae; ++e) {
      const int k = __ldg(p.colA + e);
      const float a = __ldg(p.valA + e);
      for (int q = __ldg(p.rpB + k) + t; q < __ldg(p.rpB + k + 1); q += GROUP) {
        const int r = pos[hash_find<TS>(keys, __ldg(p.colB + q))];
        acc[r] = fmaf(a, __ldg(p.valB + q), acc[r]);
      }
      group_sync<GROUP>();
    }
    for (int r = t; r < c; r += GROUP) p.valC[base + r] = acc[r];
    group_sync<GROUP>();
  }
}

struct NoSort {};

template <bool FILL>
__global__ void __launch_bounds__(SPG_WARPS * 32) spg_warp_kernel(const SpgParams p) {
  extern __shared__ __align__(16) int smem[];
  constexpr int TS = 2 * SPG_WARP_CAP;
  const int w = threadIdx.x >> 5;
  int *keys = smem + w * (2 * TS + SPG_WARP_CAP + 1);
  int *pos = keys + TS;
  float *acc = reinterpret_cast<float *>(pos + TS);
  int *ctr = pos + TS + SPG_WARP_CAP;
  const int n_rows = __ldcg(p.list_n + 0);
  for (int li = blockIdx.x * SPG_WARPS + w; li < n_rows; li += gridDim.x * SPG_WARPS)
    hash_row<32, SPG_WARP_CAP, FILL, NoSort>(p, __ldcg(p.lists + li), threadIdx.x & 31, keys, pos, acc, ctr, nullptr);
}

template <bool FILL>
__global__ void __launch_bounds__(SPG_BLOCK_THREADS) spg_block_kernel(const SpgParams p) {
  using Sort = cub::BlockRadixSort<int, SPG_BLOCK_THREADS, SPG_BLOCK_CAP / SPG_BLOCK_THREADS>;
  __shared__ typename Sort::TempStorage sort_tmp;
  __shared__ int ctr;
  extern __shared__ __align__(16) int smem[];
  constexpr int TS = 2 * SPG_BLOCK_CAP;
  int *keys = smem, *pos = smem + TS;
  float *acc = reinterpret_cast<float *>(smem + 2 * TS);
  const int n_rows = __ldcg(p.list_n + 1);
  for (int li = blockIdx.x; li < n_rows; li += gridDim.x)
    hash_row<SPG_BLOCK_THREADS, SPG_BLOCK_CAP, FILL>(p, __ldcg(p.lists + (int64_t)p.m + li), threadIdx.x, keys, pos, acc, &ctr,
                                                     &sort_tmp);
}

// Rows beyond the block tier: a bitmap of the n output columns in this block's slice of global scratch.  Threads of a
// warp that set bits of one word OR them together first (B rows are sorted, so they are neighbours) and one atomicOr
// per word goes to L2.  Scratch is read with ld.cg: the atomics are performed at L2.
template <bool FILL>
__global__ void __launch_bounds__(SPG_BLOCK_THREADS) spg_large_kernel(const SpgParams p) {
  using Scan = cub::BlockScan<int, SPG_BLOCK_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ long long total;
  unsigned *bits = p.bits + (int64_t)blockIdx.x * p.words;
  int *wp = p.wordpos + (int64_t)blockIdx.x * p.words;
  const int t = threadIdx.x, lane = t & 31;
  const int n_rows = __ldcg(p.list_n + 2);
  if ((int)blockIdx.x < n_rows) {   // the slot is zeroed here, only by blocks that have rows, and after every row
    for (int w = t; w < p.words; w += SPG_BLOCK_THREADS) __stcg(bits + w, 0u);
    __syncthreads();
  }
  for (int li = blockIdx.x; li < n_rows; li += gridDim.x) {
    const int row = __ldcg(p.lists + 2 * (int64_t)p.m + li);
    const int ab = __ldg(p.rpA + row), ae = __ldg(p.rpA + row + 1);
    for (int e = ab; e < ae; ++e) {
      const int k = __ldg(p.colA + e);
      const int bb = __ldg(p.rpB + k), be = __ldg(p.rpB + k + 1);
      for (int q0 = bb; q0 < be; q0 += SPG_BLOCK_THREADS) {
        const int q = q0 + t;
        const int j = q < be ? __ldg(p.colB + q) : -1;
        const int w = j >> 5;
        unsigned bit = q < be ? 1u << (j & 31) : 0u;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {   // segmented suffix OR over the lanes of one word
          const unsigned ob = __shfl_down_sync(FULL, bit, off);
          const int ow = __shfl_down_sync(FULL, w, off);
          if (lane + off < 32 && ow == w) bit |= ob;
        }
        const int pw = __shfl_up_sync(FULL, w, 1);
        if (q < be && (lane == 0 || pw != w)) atomicOr(bits + w, bit);
      }
    }
    __syncthreads();
    if constexpr (!FILL) {
      if (t == 0) total = 0;
      __syncthreads();
      long long mine = 0;
      for (int w = t; w < p.words; w += SPG_BLOCK_THREADS) {
        mine += __popc(__ldcg(bits + w));
        __stcg(bits + w, 0u);
      }
      if (mine) atomicAdd(reinterpret_cast<unsigned long long *>(&total), (unsigned long long)mine);
      __syncthreads();
      if (t == 0) p.cnt[row] = total;
      __syncthreads();
    } else {
      const int base = __ldg(p.rpC + row);
      int carry = 0;
      for (int w0 = 0; w0 < p.words; w0 += SPG_BLOCK_THREADS) {
        const int w = w0 + t;
        const int v = w < p.words ? __popc(__ldcg(bits + w)) : 0;
        int ex, tile;
        Scan(scan_tmp).ExclusiveSum(v, ex, tile);
        if (w < p.words) __stcg(wp + w, carry + ex);
        carry += tile;
        __syncthreads();
      }
      for (int w = t; w < p.words; w += SPG_BLOCK_THREADS) {
        unsigned b = __ldcg(bits + w);
        int r = base + __ldcg(wp + w);
        while (b) {
          __stcg(p.colC + r, w * 32 + __ffs(b) - 1);
          __stcg(p.valC + r, 0.f);
          ++r;
          b &= b - 1;
        }
      }
      __syncthreads();
      for (int e = ab; e < ae; ++e) {
        const int k = __ldg(p.colA + e);
        const float a = __ldg(p.valA + e);
        for (int q = __ldg(p.rpB + k) + t; q < __ldg(p.rpB + k + 1); q += SPG_BLOCK_THREADS) {
          const int j = __ldg(p.colB + q), w = j >> 5;
          const int r = base + __ldcg(wp + w) + __popc(__ldcg(bits + w) & ((1u << (j & 31)) - 1u));
          __stcg(p.valC + r, fmaf(a, __ldg(p.valB + q), __ldcg(p.valC + r)));
        }
        __syncthreads();
      }
      for (int w = t; w < p.words; w += SPG_BLOCK_THREADS) __stcg(bits + w, 0u);
      __syncthreads();
    }
  }
}

// largest r in [0, n] with rp[r] <= e: the row owning CSR position e
__device__ __forceinline__ int row_of(const int *__restrict__ rp, int n, int e) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(rp + mid) <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// position of column j in C's sorted row [cb, ce) (present by construction)
__device__ __forceinline__ int find_col(const int *__restrict__ colC, int cb, int ce, int j) {
  int lo = cb, hi = ce - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(colC + mid) < j) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct SpgBwdParams {
  const int *rpA, *colA;
  const float *valA;
  const int *rpB, *colB;
  const float *valB;
  const int *rpC, *colC;
  const float *dC;
  const int *colptrAT, *rowindAT, *permAT;
  float *dA, *dB;
  int m, kb;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(FULL, v, off);
  return v;
}

__global__ void spg_dA_kernel(const SpgBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int nnz = __ldg(p.rpA + p.m);
  for (int64_t e = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < nnz; e += nw) {
    const int i = row_of(p.rpA, p.m, (int)e), k = __ldg(p.colA + e);
    const int cb = __ldg(p.rpC + i), ce = __ldg(p.rpC + i + 1);
    float acc = 0.f;
    for (int q = __ldg(p.rpB + k) + lane; q < __ldg(p.rpB + k + 1); q += 32)
      acc = fmaf(__ldg(p.valB + q), __ldg(p.dC + find_col(p.colC, cb, ce, __ldg(p.colB + q))), acc);
    acc = warp_sum(acc);
    if (lane == 0) p.dA[e] = acc;
  }
}

__global__ void spg_dB_kernel(const SpgBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int nnz = __ldg(p.rpB + p.kb);
  for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nnz; q += nw) {
    const int k = row_of(p.rpB, p.kb, (int)q), j = __ldg(p.colB + q);
    float acc = 0.f;
    for (int s = __ldg(p.colptrAT + k) + lane; s < __ldg(p.colptrAT + k + 1); s += 32) {
      const int i = __ldg(p.rowindAT + s);
      acc = fmaf(__ldg(p.valA + __ldg(p.permAT + s)),
                 __ldg(p.dC + find_col(p.colC, __ldg(p.rpC + i), __ldg(p.rpC + i + 1), j)), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) p.dB[q] = acc;
  }
}

static inline int64_t al256(int64_t x) { return (x + 255) & ~(int64_t)255; }

static int64_t scan_temp_bytes(int64_t items) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const long long *)nullptr, (long long *)nullptr, (int)items);
  return (int64_t)bytes;
}

static int64_t words_for(int64_t n) { return (n + 31) / 32; }

constexpr size_t SPG_WARP_SMEM = (size_t)SPG_WARPS * (4 * SPG_WARP_CAP + SPG_WARP_CAP + 1) * sizeof(int);
constexpr size_t SPG_BLOCK_SMEM = (size_t)(4 * SPG_BLOCK_CAP + SPG_BLOCK_CAP) * sizeof(int);

// Validates the shapes shared by every entry point; `who` names the caller in the message.
static int check_shapes(const char *who, const void *rpA, const void *colA, int64_t a_rows, int64_t a_cols,
                        const void *rpB, const void *colB, int64_t b_rows, int64_t b_cols) {
  CB_REQUIRE(a_rows >= 0 && a_cols >= 0 && b_rows >= 0 && b_cols >= 0, "%s: negative size", who);
  CB_REQUIRE(rpA && colA && rpB && colB, "%s: null pointer", who);
  CB_REQUIRE(b_rows == a_cols, "%s: B has %lld rows, A has %lld columns", who, (long long)b_rows, (long long)a_cols);
  CB_REQUIRE(a_rows < 0x7fffffffLL && a_cols < 0x7fffffffLL && b_cols < 0x7fffffffLL, "%s: sizes must fit int32", who);
  return COGDL_B200_OK;
}

struct SpgScratch {
  int *list_n, *lists;
  long long *cnt, *scan;
  void *scan_tmp;
  size_t scan_tmp_bytes;
  unsigned *bits;
  int *wordpos;
};

static SpgScratch carve(void *scratch, int64_t m, int64_t n) {
  char *s = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(scratch) + 255) & ~(uintptr_t)255);
  SpgScratch r;
  r.list_n = reinterpret_cast<int *>(s); s += 256;
  r.lists = reinterpret_cast<int *>(s); s += al256(3 * m * 4);
  r.cnt = reinterpret_cast<long long *>(s); s += al256((m + 1) * 8);
  r.scan = reinterpret_cast<long long *>(s); s += al256((m + 1) * 8);
  r.scan_tmp_bytes = (size_t)scan_temp_bytes(m + 1);
  r.scan_tmp = s; s += al256((int64_t)r.scan_tmp_bytes);
  const int64_t slot_bytes = al256(SPG_LARGE_SLOTS * words_for(n) * 4);
  r.bits = reinterpret_cast<unsigned *>(s); s += slot_bytes;
  r.wordpos = reinterpret_cast<int *>(s);
  return r;
}

static unsigned capped_grid(int64_t want, int64_t cap) {
  return (unsigned)(want < 1 ? 1 : want > cap ? cap : want);
}

// classify + the three tier kernels of one phase
template <bool FILL>
static int run_tiers(SpgParams &prm, const SpgScratch &sc, int64_t m, cudaStream_t s) {
  static unsigned long long attr_done = 0;
  int dev = 0;
  if (first_use_on_device(attr_done, &dev)) {
    CB_CUDA(cudaFuncSetAttribute(spg_warp_kernel<FILL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SPG_WARP_SMEM));
    CB_CUDA(cudaFuncSetAttribute(spg_block_kernel<FILL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SPG_BLOCK_SMEM));
  }
  CB_CUDA(cudaMemsetAsync(sc.list_n, 0, 3 * sizeof(int), s));
  spg_classify_kernel<<<capped_grid(ceil_div(m, 8), NUM_SMS * 16), 256, 0, s>>>(prm, !FILL);
  CB_LAUNCH_CHECK();
  spg_warp_kernel<FILL><<<capped_grid(ceil_div(m, SPG_WARPS), NUM_SMS * 8), SPG_WARPS * 32, SPG_WARP_SMEM, s>>>(prm);
  CB_LAUNCH_CHECK();
  spg_block_kernel<FILL><<<capped_grid(m, NUM_SMS * 2), SPG_BLOCK_THREADS, SPG_BLOCK_SMEM, s>>>(prm);
  CB_LAUNCH_CHECK();
  spg_large_kernel<FILL><<<capped_grid(m, SPG_LARGE_SLOTS), SPG_BLOCK_THREADS, 0, s>>>(prm);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

static SpgParams make_params(const int32_t *rpA, const int32_t *colA, const float *valA, const int32_t *rpB,
                             const int32_t *colB, const float *valB, int64_t m, int64_t n, const SpgScratch &sc) {
  SpgParams prm;
  prm.rpA = rpA; prm.colA = colA; prm.valA = valA;
  prm.rpB = rpB; prm.colB = colB; prm.valB = valB;
  prm.m = (int)m; prm.n = (int)n; prm.words = (int)words_for(n);
  prm.rpC = nullptr; prm.colC = nullptr; prm.valC = nullptr;
  prm.cnt = sc.cnt; prm.lists = sc.lists; prm.list_n = sc.list_n;
  prm.bits = sc.bits; prm.wordpos = sc.wordpos;
  return prm;
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_spgemm_scratch_bytes(int64_t a_rows, int64_t a_cols, int64_t b_cols) {
  (void)a_cols;
  if (a_rows < 0 || b_cols < 0) return -1;
  const int64_t m = a_rows;
  return 256 + 256 + al256(3 * m * 4) + 2 * al256((m + 1) * 8) + al256(scan_temp_bytes(m + 1)) +
         2 * al256(SPG_LARGE_SLOTS * words_for(b_cols) * 4);
}

extern "C" int cogdl_b200_spgemm_count(const int32_t *rowptrA, const int32_t *colA, int64_t a_rows, int64_t a_cols,
                                       const int32_t *rowptrB, const int32_t *colB, int64_t b_rows, int64_t b_cols,
                                       int32_t *rowptrC, int64_t *nnz_c, void *scratch, int64_t scratch_bytes,
                                       cogdl_b200_stream_t stream) {
  int rc = check_shapes("cogdl_b200_spgemm_count", rowptrA, colA, a_rows, a_cols, rowptrB, colB, b_rows, b_cols);
  if (rc) return rc;
  CB_REQUIRE(rowptrC && nnz_c && scratch, "cogdl_b200_spgemm_count: null pointer");
  CB_REQUIRE(scratch_bytes >= cogdl_b200_spgemm_scratch_bytes(a_rows, a_cols, b_cols),
             "cogdl_b200_spgemm_count: scratch too small (%lld bytes, need %lld)", (long long)scratch_bytes,
             (long long)cogdl_b200_spgemm_scratch_bytes(a_rows, a_cols, b_cols));
  cudaStream_t s = (cudaStream_t)stream;
  note_kernel("cogdl_b200::spg_count<warp=%d,block=%d,bitmap>", SPG_WARP_CAP, SPG_BLOCK_CAP);
  const int64_t m = a_rows;
  if (m == 0) {
    CB_CUDA(cudaMemsetAsync(rowptrC, 0, sizeof(int32_t), s));
    *nnz_c = 0;
    return COGDL_B200_OK;
  }
  const SpgScratch sc = carve(scratch, m, b_cols);
  SpgParams prm = make_params(rowptrA, colA, nullptr, rowptrB, colB, nullptr, m, b_cols, sc);
  rc = run_tiers<false>(prm, sc, m, s);
  if (rc) return rc;
  CB_CUDA(cudaMemsetAsync(sc.cnt + m, 0, sizeof(long long), s));
  size_t tmp = sc.scan_tmp_bytes;
  CB_CUDA(cub::DeviceScan::ExclusiveSum(sc.scan_tmp, tmp, sc.cnt, sc.scan, (int)(m + 1), s));
  count_launch();
  long long total = 0;
  CB_CUDA(cudaMemcpyAsync(&total, sc.scan + m, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CB_CUDA(cudaStreamSynchronize(s));
  CB_REQUIRE(total <= 0x7fffffffLL, "cogdl_b200_spgemm_count: the product has %lld entries, more than int32 CSR holds",
             total);
  *nnz_c = total;
  return cogdl_b200_narrow_i64_i32(reinterpret_cast<const int64_t *>(sc.scan), rowptrC, m + 1, stream);
}

extern "C" int cogdl_b200_spgemm_fill_f32(const int32_t *rowptrA, const int32_t *colA, const float *valA, int64_t a_rows,
                                          int64_t a_cols, const int32_t *rowptrB, const int32_t *colB, const float *valB,
                                          int64_t b_rows, int64_t b_cols, const int32_t *rowptrC, int32_t *colC,
                                          float *valC, void *scratch, int64_t scratch_bytes,
                                          cogdl_b200_stream_t stream) {
  int rc = check_shapes("cogdl_b200_spgemm_fill_f32", rowptrA, colA, a_rows, a_cols, rowptrB, colB, b_rows, b_cols);
  if (rc) return rc;
  CB_REQUIRE(valA && valB && rowptrC && colC && valC && scratch, "cogdl_b200_spgemm_fill_f32: null pointer");
  CB_REQUIRE(scratch_bytes >= cogdl_b200_spgemm_scratch_bytes(a_rows, a_cols, b_cols),
             "cogdl_b200_spgemm_fill_f32: scratch too small (%lld bytes, need %lld)", (long long)scratch_bytes,
             (long long)cogdl_b200_spgemm_scratch_bytes(a_rows, a_cols, b_cols));
  note_kernel("cogdl_b200::spg_fill<warp=%d,block=%d,bitmap>", SPG_WARP_CAP, SPG_BLOCK_CAP);
  const int64_t m = a_rows;
  if (m == 0) return COGDL_B200_OK;
  const SpgScratch sc = carve(scratch, m, b_cols);
  SpgParams prm = make_params(rowptrA, colA, valA, rowptrB, colB, valB, m, b_cols, sc);
  prm.rpC = rowptrC; prm.colC = colC; prm.valC = valC;
  return run_tiers<true>(prm, sc, m, (cudaStream_t)stream);
}

extern "C" int cogdl_b200_spgemm_bwd_f32(const int32_t *rowptrA, const int32_t *colA, const float *valA, int64_t a_rows,
                                         int64_t a_cols, const int32_t *rowptrB, const int32_t *colB, const float *valB,
                                         int64_t b_rows, int64_t b_cols, const int32_t *rowptrC, const int32_t *colC,
                                         const float *dC, const int32_t *colptrAT, const int32_t *rowindAT,
                                         const int32_t *permAT, float *dA, float *dB, cogdl_b200_stream_t stream) {
  int rc = check_shapes("cogdl_b200_spgemm_bwd_f32", rowptrA, colA, a_rows, a_cols, rowptrB, colB, b_rows, b_cols);
  if (rc) return rc;
  CB_REQUIRE(rowptrC && colC && dC, "cogdl_b200_spgemm_bwd_f32: null pointer");
  CB_REQUIRE(!dA || valB, "cogdl_b200_spgemm_bwd_f32: dA needs valB");
  CB_REQUIRE(!dB || (valA && colptrAT && rowindAT && permAT), "cogdl_b200_spgemm_bwd_f32: dB needs valA and A's transpose");
  SpgBwdParams p;
  p.rpA = rowptrA; p.colA = colA; p.valA = valA; p.rpB = rowptrB; p.colB = colB; p.valB = valB;
  p.rpC = rowptrC; p.colC = colC; p.dC = dC;
  p.colptrAT = colptrAT; p.rowindAT = rowindAT; p.permAT = permAT;
  p.dA = dA; p.dB = dB; p.m = (int)a_rows; p.kb = (int)b_rows;
  cudaStream_t s = (cudaStream_t)stream;
  if (dA) {
    note_kernel("cogdl_b200::spg_dA_kernel");
    spg_dA_kernel<<<NUM_SMS * 16, 256, 0, s>>>(p);
    CB_LAUNCH_CHECK();
  }
  if (dB) {
    note_kernel(dA ? "cogdl_b200::spg_dA_kernel + cogdl_b200::spg_dB_kernel" : "cogdl_b200::spg_dB_kernel");
    spg_dB_kernel<<<NUM_SMS * 16, 256, 0, s>>>(p);
    CB_LAUNCH_CHECK();
  }
  return COGDL_B200_OK;
}

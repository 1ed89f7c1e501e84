// fused_gcn.cu -- GCN layer with the dense transform fused onto the aggregated tile (SURVEY 8f-3):
//
//     OUT[i,:] = act( (sum_p val[p] * X[col[p],:]) . W^T  +  (sum_p val[p]) * b )          i.e.  (A.X).W^T + (A.1) b^T
//
// which equals the reference's  A.(X.W^T + 1 b^T)  (cogdl/layers/gcn_layer.py:51-64: `support = self.linear(x);
// out = spmm(graph, support)`; bias INSIDE the aggregation, then activation) up to fp32 rounding -- the order of
// the two products is swapped so that the sparse gather runs on the raw features and the GEMM runs on the
// aggregated 128-row tile while it is still on chip.  Behind a flag in the Python layer because it reorders.
// This is the only tensor-core work on the hot path (north star: "tensor cores only where a dense
// feature x weight GEMM is fused onto the aggregated output").
//
// One persistent CTA per SM made of TWO independent 8-warp groups; each group owns a tile of 64 consecutive
// destination rows (its own operand buffer and named barrier) and both share W^T.  The groups drift apart by
// construction, so while one waits for its tensor-core products and writes its output the other keeps the SM's
// load pipeline busy.
//   1. AGGREGATE (the group's warps): the tile's rows are dealt to the warps in contiguous runs of ~equal COST
//      (rowptr of the tile staged one tile ahead); each warp streams the edges of its rows like the row-stream SpMM
//      (stream.cuh: 32-edge slabs, ballot row-end masks, U independent 512-byte gathers in flight, CSR order
//      with separate fp32 mul / add => the aggregated tile is bit-identical to the SpMM output).  At a row end
//      the fp32 row is NOT stored to global memory: it is split into three bf16 terms a = a1 + a2 + a3
//      (a1 = bf16(a), a2 = bf16(a - a1), a3 = bf16(a - a1 - a2): 24 mantissa bits) and written into shared memory
//      in the wgmma K-major SWIZZLE_128B operand layout.  Hub rows (degree > plan chunk) were aggregated
//      beforehand by the hub-chunk items of the row-stream kernel (deterministic in-order combine) and are
//      picked up from a scratch matrix.
//   2. MMA (the group's two warpgroups, one 64-column half of the output each, in two 32-column passes; passes
//      at or beyond Fout are skipped): D[64 x 32] (fp32, registers) = sum over the six split products a_i . w_j with
//      i + j <= 4 (a3.w1, a2.w2, a1.w3, a2.w1, a1.w2, a1.w1 -- small terms first), each 8 x wgmma.mma_async
//      m64n32k16 bf16 of K = 16, both operands read from shared memory, W^T resident there (split the same way
//      once per CTA).
//      Dropped terms are <= 2^-24 relative: error vs an fp64 product ~1e-7 of the row scale, i.e. better than
//      an fp32 FFMA GEMM (TF32 would give 1e-3, plain bf16 4e-3; tests/test_cpu_oracle_and_host.py emulates the
//      split in numpy).
//   3. EPILOGUE (the same warpgroup, after each pass): add rowsum * bias to the accumulator registers, ReLU, store.
// No reference counterpart as a kernel; callers cogdl/layers/gcn_layer.py:51-64 (and sage_layer.py:69-87 for the
// aggregate-then-linear order).  K (input width) must be 128, Fout <= 128.
//
// GraphSAGE form (cogdl/layers/sage_layer.py:69-87, fc(cat[x, agg]) with fc.weight = [W_self | W_neigh]):
//     OUT[i,:] = act( S[i,:] + agg_i(X) . W_neigh^T ),   S = X[:n] . W_self^T + b   (library GEMM, beforehand)
// The same kernel, templated on the aggregation (AGG) and on the epilogue addend (EPI):
//   AGG_SUM  the gather above, optionally times a per-row fp32 scale (graph.in_norm of a CSR-only graph, applied
//            to the fp32 row before the split, hub rows included: bit-identical to `in_norm * spmm(...)`);
//            mean is SUM with row-normalised edge weights or with that scale;
//   AGG_MAX  running max from -inf with the strict `<` update of scatter_max.cu, degree-0 rows 0 (bit-identical to
//            scatter_max_fwd's values; no argmax: the backward recomputes it).  Hub rows come from a pre-pass of
//            scatter_max's row-stream kernel (hub chunks only, argmax stores compiled out);
//   EPI_BIAS add rowsum * bias (GCN);  EPI_SELF add S[row, c] (SAGE).
// The self half is not put on the tensor cores: a bf16x3 W^T for K = 256 takes 192 KB, and the two 48 KB operand
// tiles do not fit beside it in the SM's 227 KB.  W_neigh ([Fout,128]) fills the 96 KB W^T buffer as W does for GCN.
#include "common.cuh"
#include "stream.cuh"

#include <cuda_bf16.h>
#include <math_constants.h>

namespace cogdl_b200 {

int spmm_hub_rows_only(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X, float *Y,
                       int64_t F, const cogdl_b200_hub_plan_t *plan, cudaStream_t stream);
int smax_hub_rows_only(const int32_t *rowptr, const int32_t *colind, const float *X, float *Y, int64_t F,
                       const cogdl_b200_hub_plan_t *plan, cudaStream_t stream);

namespace fg {

enum { AGG_SUM = 0, AGG_MAX = 1 };
enum { EPI_BIAS = 0, EPI_SELF = 1 };

constexpr int TILE_M = 64;                            // rows per tile (wgmma M = 64); two tiles are in flight per CTA
constexpr int GROUPS = 2;                             // independent warp groups, one tile each, W^T shared
constexpr int GWARPS = 8;                             // warps per group
constexpr int WARPS = GROUPS * GWARPS;
constexpr int KDIM = 128;
constexpr int U = 8;                                  // gathers per batch; two batches in flight per warp (software pipelined):
                                                      // 16 warps x 16 x 512 B = 128 KB of feature rows in flight per SM
constexpr int SLAB_BYTES_A = TILE_M * 128;            // one K-slab (64 bf16 = 128 B per row) of a tile: 8 KB
constexpr int A_TILE_BYTES = 3 * 2 * SLAB_BYTES_A;    // 3 splits x 2 K-slabs = 48 KB per group
constexpr int WG_N = 64;                              // output columns per warpgroup
constexpr int WG_NP = 32;                             // columns per MMA pass (wgmma N)
constexpr int W_SLAB_BYTES = 128 * 128;              // one K-slab of W^T, laid out for 128 rows whatever Fout
constexpr int W_MAX_BYTES = 3 * 2 * W_SLAB_BYTES;     // 96 KB
constexpr int OFF_W = GROUPS * A_TILE_BYTES;
constexpr int OFF_BIAS = OFF_W + W_MAX_BYTES;
constexpr int OFF_GROUP = OFF_BIAS + 128 * 4;         // per group: rowsum[64] | tile_rp[68] | tile_cost[68]
constexpr int GROUP_BYTES = TILE_M * 4 + 2 * (TILE_M + 4) * 4;
constexpr int OFF_SLAB = OFF_GROUP + GROUPS * GROUP_BYTES;      // per warp: 32 x (column, value) + 32 x row
constexpr int SMEM_BYTES = OFF_SLAB + WARPS * 32 * 12 + 1024;   // + slack to align the base to 1024 B (SWIZZLE_128B atoms)

struct Params {
  const int *rowptr;
  const int *colind;
  const float *val;        // nullable
  const int *edge_row;     // plan->edge_row
  const float *X;          // [n_src, 128]
  const float *W;          // [Fout, 128]  (nn.Linear weight layout = K-major B operand)
  const float *bias;       // nullable [Fout]
  const float *hub_agg;    // [n_rows, 128]: rows with degree > chunk_edges hold (A.X)[row]
  const float *rowsum;     // nullable [n_rows]: (A.1)[row], cached by the caller for fixed edge weights
  float *out;              // [n_rows, Fout]
  int n_rows;
  int Fout;
  int Npad;                // rows of W^T filled in shared memory: 64 if Fout <= 64, else 128 (zero-padded)
  int chunk_edges;         // 0: no hub rows anywhere
  int relu;
  int n_tiles;
  // EPI_SELF only (appended so the fields above keep their offsets)
  const float *row_scale;  // nullable [n_rows]: multiplies the aggregated row (AGG_SUM)
  const float *S;          // [n_rows, Fout]: epilogue addend
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void group_sync(int g) {     // named barrier of one warp group (ids 1, 2; 0 is __syncthreads)
  asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "r"(GWARPS * 32) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from touching an accumulator register across an asynchronous wgmma
__device__ __forceinline__ void fence_operand(float &r) { asm volatile("" : "+f"(r)::"memory"); }
// D[64 x 32] (+)= A[smem desc] . B[smem desc]^T, bf16 inputs, fp32 accumulate, issued by all 128 threads of a warpgroup.
// Fragment of thread (warp w of the warpgroup, lane l): d[4j + 2i + c] = D[16w + l/4 + 8i][8j + 2(l%4) + c].
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t desc_a, uint64_t desc_b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// Feature-row gathers bypass the L1: this kernel leaves the SM ~28 KB of L1 (228 KB shared-memory carve-out), and an L1-allocating
// load holds a line per 128 bytes in flight -- 128 lines cap the SM at ~32 row gathers in flight, whatever the warp count
// or unroll depth (measured: three different schedules all landed on the same time).  ld.global.cg is tracked outside the
// L1 data array.
__device__ __forceinline__ float4 fg_gather(const float4 *p) { return __ldcg(p); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (PTX ISA "Matrix Descriptor Format"):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024 B between 8-row groups) | [49,52) base offset = 0
//   [62,64) layout type = 1 (SWIZZLE_128B).  Every 8-row group starts 1024-byte aligned; a K step of 16 inside the
//   128-byte swizzle atom advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// byte offset of bf16 element (row r, k) inside one split of a [rows x 128] K-major SW128 operand whose K-slabs
// (64 elements = 128 B per row) are `slab_bytes` apart
__device__ __forceinline__ uint32_t sw128_offset(int r, int k, int slab_bytes) {
  const int slab = k >> 6, kk = k & 63;
  const int chunk = (kk >> 3) ^ (r & 7);
  return (uint32_t)(slab * slab_bytes + (r >> 3) * 1024 + (r & 7) * 128 + chunk * 16 + (kk & 7) * 2);
}

// a = a1 + a2 + a3 (bf16 each, round to nearest even; the residuals are exact in fp32).  A finite a that rounds to
// a bf16 infinity (|a| >= 0x1.fefp127) is rounded toward zero instead, so its residual stays finite; a non-finite a
// goes whole into a1 with zero residuals (a - bf16(a) would be Inf - Inf = NaN).
__device__ __forceinline__ void split3(float a, __nv_bfloat16 &a1, __nv_bfloat16 &a2, __nv_bfloat16 &a3) {
  a1 = __float2bfloat16_rn(a);
  if (__hisinf(a1) && isfinite(a)) a1 = __float2bfloat16_rz(a);
  const float r1 = isfinite(a) ? a - __bfloat162float(a1) : 0.f;
  a2 = __float2bfloat16_rn(r1);
  const float r2 = r1 - __bfloat162float(a2);
  a3 = __float2bfloat16_rn(r2);
}
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 lo, __nv_bfloat16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// write one aggregated row (lane owns columns 4*lane .. 4*lane+3) into the three split operands of a tile
__device__ __forceinline__ void store_row(unsigned char *tileA, int r, int lane, const float4 &acc) {
  __nv_bfloat16 s1[4], s2[4], s3[4];
  split3(acc.x, s1[0], s2[0], s3[0]);
  split3(acc.y, s1[1], s2[1], s3[1]);
  split3(acc.z, s1[2], s2[2], s3[2]);
  split3(acc.w, s1[3], s2[3], s3[3]);
  const uint32_t off = sw128_offset(r, 4 * lane, SLAB_BYTES_A);
  *reinterpret_cast<uint2 *>(tileA + 0 * 2 * SLAB_BYTES_A + off) = make_uint2(pack2(s1[0], s1[1]), pack2(s1[2], s1[3]));
  *reinterpret_cast<uint2 *>(tileA + 1 * 2 * SLAB_BYTES_A + off) = make_uint2(pack2(s2[0], s2[1]), pack2(s2[2], s2[3]));
  *reinterpret_cast<uint2 *>(tileA + 2 * 2 * SLAB_BYTES_A + off) = make_uint2(pack2(s3[0], s3[1]), pack2(s3[2], s3[3]));
}

// AGG_MAX accumulator: strict `<` as scatter_max.cu (first value wins ties, a NaN never replaces the running max)
__device__ __forceinline__ void max_upd(float4 &m, const float4 &x) {
  if (m.x < x.x) m.x = x.x;
  if (m.y < x.y) m.y = x.y;
  if (m.z < x.z) m.z = x.z;
  if (m.w < x.w) m.w = x.w;
}
template <int AGG> __device__ __forceinline__ float4 agg_init() {
  return AGG == AGG_MAX ? make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
}
// the row scale as `in_norm * x` applies it: one rounded product (never contracted into the split's subtractions)
__device__ __forceinline__ float4 scale_row(const float4 &a, float s) {
  return make_float4(__fmul_rn(s, a.x), __fmul_rn(s, a.y), __fmul_rn(s, a.z), __fmul_rn(s, a.w));
}

// rowptr and cost prefix of one 64-row tile -> shared memory (one warp: lane L takes rows 2L, 2L+1).  cost(row) =
// 1 + (hub ? 4 : deg): hub rows are one 512-byte read here, their edges were consumed by the hub pre-pass
__device__ __forceinline__ void stage_tile(const Params &p, int row0, int lane, int *tile_rp, int *tile_cost) {
  int rp[3];
#pragma unroll
  for (int t = 0; t < 3; ++t) rp[t] = __ldg(p.rowptr + min(row0 + 2 * lane + t, p.n_rows));
  int c[2], tot = 0;
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int d = rp[t + 1] - rp[t];
    c[t] = (row0 + 2 * lane + t < p.n_rows) ? 1 + ((p.chunk_edges > 0 && d > p.chunk_edges) ? 4 : d) : 0;
    tot += c[t];
  }
  int incl = tot;
#pragma unroll
  for (int st = 1; st < 32; st <<= 1) {
    const int o = __shfl_up_sync(FULL, incl, st);
    if (lane >= st) incl += o;
  }
  int run = incl - tot;
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    tile_rp[2 * lane + t] = rp[t];
    tile_cost[2 * lane + t] = run;
    run += c[t];
  }
  if (lane == 31) { tile_rp[TILE_M] = rp[2]; tile_cost[TILE_M] = run; }
}

template <int AGG, int EPI>
__global__ void __launch_bounds__(WARPS * 32, 1) fused_layer_kernel(const Params p) {
  extern __shared__ unsigned char fg_smem_raw[];
  // SWIZZLE_128B atoms need a 1024-byte aligned base
  unsigned char *smem = fg_smem_raw + ((1024u - (smem_u32(fg_smem_raw) & 1023u)) & 1023u);   // stays a shared-space pointer
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = warp / GWARPS, gw = warp % GWARPS;   // my group, warp inside it
  unsigned char *tileA = smem + g * A_TILE_BYTES;
  unsigned char *smemW = smem + OFF_W;
  float *bias_s = reinterpret_cast<float *>(smem + OFF_BIAS);
  unsigned char *gbase = smem + OFF_GROUP + g * GROUP_BYTES;
  float *rowsum_s = reinterpret_cast<float *>(gbase);
  int *tile_rp = reinterpret_cast<int *>(gbase + TILE_M * 4);
  int *tile_cost = tile_rp + (TILE_M + 4);
  int2 *s_cv = reinterpret_cast<int2 *>(smem + OFF_SLAB) + warp * 32;
  int *s_r = reinterpret_cast<int *>(smem + OFF_SLAB + WARPS * 32 * 8) + warp * 32;
  const int tile_stride = (int)gridDim.x * GROUPS;
  const int first_tile = (int)blockIdx.x * GROUPS + g;

  // ---- one-time setup: W^T split into three bf16 operands (SW128 K-major, rows >= Fout zero), bias
  for (int idx = tid; idx < p.Npad * (KDIM / 4); idx += WARPS * 32) {     // 4 consecutive k per thread
    const int n = idx / (KDIM / 4), k = (idx - n * (KDIM / 4)) * 4;
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < p.Fout) w = __ldg(reinterpret_cast<const float4 *>(p.W + (int64_t)n * KDIM + k));
    __nv_bfloat16 s1[4], s2[4], s3[4];
    split3(w.x, s1[0], s2[0], s3[0]);
    split3(w.y, s1[1], s2[1], s3[1]);
    split3(w.z, s1[2], s2[2], s3[2]);
    split3(w.w, s1[3], s2[3], s3[3]);
    const uint32_t off = sw128_offset(n, k, W_SLAB_BYTES);
    *reinterpret_cast<uint2 *>(smemW + 0 * 2 * W_SLAB_BYTES + off) = make_uint2(pack2(s1[0], s1[1]), pack2(s1[2], s1[3]));
    *reinterpret_cast<uint2 *>(smemW + 1 * 2 * W_SLAB_BYTES + off) = make_uint2(pack2(s2[0], s2[1]), pack2(s2[2], s2[3]));
    *reinterpret_cast<uint2 *>(smemW + 2 * 2 * W_SLAB_BYTES + off) = make_uint2(pack2(s3[0], s3[1]), pack2(s3[2], s3[3]));
  }
  if (tid < 128) bias_s[tid] = (p.bias && tid < p.Fout) ? __ldg(p.bias + tid) : 0.f;
  if (gw == 1 && first_tile < p.n_tiles) stage_tile(p, first_tile * TILE_M, lane, tile_rp, tile_cost);
  fence_async_smem();
  __syncthreads();
  // warpgroup h (warps 4h .. 4h+3 of the group) owns output columns [64 h, 64 h + 64); its warp wq rows 16 wq .. 16 wq + 15
  const int h = gw >> 2, wq = gw & 3;
  const float4 *X4 = reinterpret_cast<const float4 *>(p.X);
  const float4 *H4 = reinterpret_cast<const float4 *>(p.hub_agg);

  // ===== the two groups run this loop independently (named barriers): while one is in its MMA / epilogue, the other
  //       keeps the SM's memory pipeline busy with its gather
  for (int tile = first_tile; tile < p.n_tiles; tile += tile_stride) {
    const int row0 = tile * TILE_M;
    // =========================================================== 1. aggregate my rows into shared memory
    // rows are dealt to the group's 8 warps by COST (contiguous runs; hub rows count as 4 edges): on power-law
    // rows an equal-rows split leaves most warps idle while one finishes (binary search in the cost prefix)
    {
      const int rows_here = min(TILE_M, p.n_rows - row0);
      const int c_tot = tile_cost[rows_here];
      auto split = [&](int w) {          // first row whose cost prefix >= share w
        if (w <= 0) return 0;
        if (w >= GWARPS) return rows_here;
        const int target = (int)(((long long)c_tot * w) / GWARPS);
        int lo = 0, hi = rows_here;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (tile_cost[mid] < target) lo = mid + 1; else hi = mid;
        }
        return lo;
      };
      const int r_begin = row0 + split(gw), r_end = row0 + split(gw + 1);
      int next_row = r_begin;      // rows < next_row of my range have been written
      auto zero_rows = [&](int upto) {   // rows [next_row, upto): no edges -> zeros
        for (; next_row < upto; ++next_row) {
          store_row(tileA, next_row - row0, lane, make_float4(0.f, 0.f, 0.f, 0.f));
          if (EPI == EPI_BIAS && lane == 0) rowsum_s[next_row - row0] = 0.f;
        }
      };
      int r = r_begin;
      while (r < r_end) {
        const int lb = tile_rp[r - row0], hb = tile_rp[r - row0 + 1];
        if (p.chunk_edges > 0 && hb - lb > p.chunk_edges) {
          // hub row: aggregated beforehand (hub chunks of the row-stream kernel)
          float4 a = __ldg(H4 + (int64_t)r * (KDIM / 4) + lane);
          float s = 0.f;
          if (EPI == EPI_SELF) {
            if (p.row_scale) a = scale_row(a, __ldg(p.row_scale + r));
          } else if (p.rowsum) {
            s = __ldg(p.rowsum + r);
          } else if (p.val) {      // no cached row sums: one warp sums the hub's weights, 8 loads in flight per lane
            float sa[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            int e = lb + lane;
            for (; e + 7 * 32 < hb; e += 256) {
#pragma unroll
              for (int t = 0; t < 8; ++t) sa[t] += ld_stream(p.val + e + 32 * t);
            }
            for (; e < hb; e += 32) sa[0] += ld_stream(p.val + e);
            s = ((sa[0] + sa[1]) + (sa[2] + sa[3])) + ((sa[4] + sa[5]) + (sa[6] + sa[7]));
            for (int st = 16; st > 0; st >>= 1) s += __shfl_xor_sync(FULL, s, st);
          } else {
            s = (float)(hb - lb);
          }
          store_row(tileA, r - row0, lane, a);
          if (EPI == EPI_BIAS && lane == 0) rowsum_s[r - row0] = s;
          next_row = r + 1;
          ++r;
          continue;
        }
        // maximal run of non-hub rows [r, rb)
        int rb = r + 1;
        while (rb < r_end && !(p.chunk_edges > 0 && tile_rp[rb - row0 + 1] - tile_rp[rb - row0] > p.chunk_edges)) ++rb;
        const int e_begin = lb, e_end = tile_rp[rb - row0];
        float4 acc = agg_init<AGG>();
        float rs = 0.f;
        auto flush = [&](int rj) {                       // last edge of row rj
          zero_rows(rj);
          if (EPI == EPI_SELF && p.row_scale) store_row(tileA, rj - row0, lane, scale_row(acc, __ldg(p.row_scale + rj)));
          else store_row(tileA, rj - row0, lane, acc);
          if (EPI == EPI_BIAS && lane == 0) rowsum_s[rj - row0] = rs;
          next_row = rj + 1;
          acc = agg_init<AGG>();
          rs = 0.f;
        };
        // slab registers (column, value, row, row of the next edge); the NEXT slab is fetched while this one is used
        int c = 0, rid = -1, rnx = -1;
        float v = 0.f;
        auto load_slab = [&](int e0, int &c_, float &v_, int &rid_, int &rnx_) {
          const int q = e0 + lane;
          c_ = 0; v_ = 0.f; rid_ = -1; rnx_ = -1;
          if (q < e_end) {
            c_ = ld_stream(p.colind + q);
            v_ = p.val ? ld_stream(p.val + q) : 1.f;
            rid_ = ld_stream(p.edge_row + q);
            if (q + 1 < e_end) rnx_ = __ldg(p.edge_row + q + 1);
          }
        };
        load_slab(e_begin, c, v, rid, rnx);
        for (int e = e_begin; e < e_end; e += 32) {
          const int cnt = min(32, e_end - e);
          const unsigned endmask = __ballot_sync(FULL, lane < cnt && rid != rnx);
          __syncwarp();                                  // previous slab fully consumed
          s_cv[lane] = make_int2(c, __float_as_int(v));  // slab parked in shared memory: broadcast LDS.64 instead of
          s_r[lane] = rid;                               // three shuffles + convergence checks per edge (stream.cuh)
          __syncwarp();
          int cn, ridn, rnxn;
          float vn;
          load_slab(e + 32, cn, vn, ridn, rnxn);
          // two batches of U gathers in flight: batch b+1 is issued before batch b is consumed
          float4 xa[U], xb[U];
          auto load_batch = [&](float4 (&x)[U], int j) {
#pragma unroll
            for (int u = 0; u < U; ++u)
              if (j + u < cnt) x[u] = fg_gather(X4 + (int64_t)s_cv[j + u].x * (KDIM / 4) + lane);
          };
          auto consume = [&](const float4 (&x)[U], int j) {
            const unsigned em = (endmask >> j) & ((1u << U) - 1u);
#pragma unroll
            for (int u = 0; u < U; ++u) {
              if (j + u < cnt) {
                const float vj = __int_as_float(s_cv[j + u].y);
                if (AGG == AGG_MAX) max_upd(acc, x[u]);
                else if (p.val) axpy_rn(acc, vj, x[u]); else add_rn(acc, x[u]);
                rs += vj;
                if (em != 0u && ((em >> u) & 1u)) flush(s_r[j + u]);
              }
            }
          };
          load_batch(xa, 0);
#pragma unroll 1
          for (int j = 0; j < cnt; j += 2 * U) {
            if (j + U < cnt) load_batch(xb, j + U);
            consume(xa, j);
            if (j + 2 * U < cnt) load_batch(xa, j + 2 * U);
            if (j + U < cnt) consume(xb, j + U);
          }
          c = cn; v = vn; rid = ridn; rnx = rnxn;
        }
        zero_rows(rb);     // trailing empty rows of the run
        r = rb;
      }
      // rows of the tile beyond n_rows (last tile): zeros, dealt round-robin
      for (int rr = rows_here + gw; rr < TILE_M; rr += GWARPS) {
        store_row(tileA, rr, lane, make_float4(0.f, 0.f, 0.f, 0.f));
        if (EPI == EPI_BIAS && lane == 0) rowsum_s[rr] = 0.f;
      }
    }
    fence_async_smem();          // generic-proxy writes of the tile -> visible to the tensor core (async proxy)
    group_sync(g);
    // rowptr + cost prefix of my NEXT tile (read again only after the barrier at the end of this tile)
    if (gw == 1 && tile + tile_stride < p.n_tiles) stage_tile(p, (tile + tile_stride) * TILE_M, lane, tile_rp, tile_cost);
    // =========================================================== 2. six split products into registers (per warpgroup)
    const uint64_t desc_a = make_desc(smem_u32(tileA));
    const bool vec = (p.Fout % 2 == 0);
    // two passes of 32 columns: 16 accumulators live at a time keep the kernel within its 128 registers
#pragma unroll 1
    for (int pass = 0; pass < WG_N / WG_NP; ++pass) {
      const int col0 = h * WG_N + pass * WG_NP;
      if (col0 >= p.Fout) break;                              // warpgroup-uniform
      const uint64_t desc_w = make_desc(smem_u32(smemW) + (uint32_t)(col0 * 128));
      // (i, j): split of A x split of W, smallest terms first: i = 2 1 0 1 0 0, j = 0 1 2 0 1 0 (one nibble per product)
      constexpr uint32_t AI = 0x001012u, WJ = 0x010210u;
      float d[WG_NP / 2];
#pragma unroll
      for (int k = 0; k < WG_NP / 2; ++k) { d[k] = 0.f; fence_operand(d[k]); }
      wgmma_fence();
      // not unrolled over the products: a fully unrolled chain keeps 48 descriptor pairs live and spills
#pragma unroll 1
      for (int t = 0; t < 6; ++t) {
        const uint32_t ai = (AI >> (4 * t)) & 0xFu, wj = (WJ >> (4 * t)) & 0xFu;
#pragma unroll
        for (int ks = 0; ks < KDIM / 16; ++ks) {            // K = 16 bf16 = 32 bytes per instruction
          // byte offsets added to the descriptors' start-address field (in 16-byte units, no carry: < 256 KB)
          const uint32_t ka = ai * 2 * SLAB_BYTES_A + (ks >> 2) * SLAB_BYTES_A + (ks & 3) * 32;
          const uint32_t kb = wj * 2 * W_SLAB_BYTES + (ks >> 2) * W_SLAB_BYTES + (ks & 3) * 32;
          wgmma_m64n32k16(d, desc_a + (ka >> 4), desc_w + (kb >> 4), (t | ks) != 0);
        }
      }
      wgmma_commit();
      // =========================================================== 3. epilogue: registers -> global
      wgmma_wait_all();
#pragma unroll
      for (int k = 0; k < WG_NP / 2; ++k) fence_operand(d[k]);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = wq * 16 + (lane >> 2) + 8 * i;
        const int grow = row0 + r;
        if (grow < p.n_rows) {
          const float rsum = EPI == EPI_BIAS ? rowsum_s[r] : 0.f;
          float *o = p.out + (int64_t)grow * p.Fout;
#pragma unroll
          for (int j = 0; j < WG_NP / 8; ++j) {
            const int c = col0 + 8 * j + 2 * (lane & 3);
            float2 y;
            if (EPI == EPI_BIAS) {
              y = make_float2(d[4 * j + 2 * i] + rsum * bias_s[c], d[4 * j + 2 * i + 1] + rsum * bias_s[c + 1]);
            } else {
              const float *srow = p.S + (int64_t)grow * p.Fout;
              float2 sv = make_float2(0.f, 0.f);
              if (vec && c + 1 < p.Fout) {
                sv = __ldcs(reinterpret_cast<const float2 *>(srow + c));
              } else {
                if (c < p.Fout) sv.x = __ldcs(srow + c);
                if (c + 1 < p.Fout) sv.y = __ldcs(srow + c + 1);
              }
              y = make_float2(d[4 * j + 2 * i] + sv.x, d[4 * j + 2 * i + 1] + sv.y);
            }
            if (p.relu) { y.x = relu_nan(y.x); y.y = relu_nan(y.y); }
            if (vec && c + 1 < p.Fout) {
              __stcs(reinterpret_cast<float2 *>(o + c), y);
            } else {
              if (c < p.Fout) o[c] = y.x;
              if (c + 1 < p.Fout) o[c + 1] = y.y;
            }
          }
        }
      }
    }
    group_sync(g);               // operand tile and staged rowptr are free / ready for the next tile
  }
}

// one persistent CTA per SM (at most one per pair of tiles)
template <int AGG, int EPI>
static int launch(const Params &p, cudaStream_t s) {
  static unsigned long long attr_done = 0;
  int dev = 0, n_sms = NUM_SMS;
  if (first_use_on_device(attr_done, &dev))
    CB_CUDA(cudaFuncSetAttribute(fused_layer_kernel<AGG, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  CB_CUDA(cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, dev));
  const int want = (p.n_tiles + GROUPS - 1) / GROUPS;
  const int grid = want < n_sms ? want : n_sms;
  fused_layer_kernel<AGG, EPI><<<grid, WARPS * 32, SMEM_BYTES, s>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

}  // namespace fg
}  // namespace cogdl_b200

using namespace cogdl_b200;

// cogdl_b200_last_kernel() of a fused layer: with hub rows, the pre-pass kernel (recorded by its launcher), " + ", then
// the fused kernel; without, the fused kernel alone
#define FG_NOTE(prepass, fmt, ...) ((prepass) ? append_kernel_note(" + " fmt, __VA_ARGS__) : note_kernel(fmt, __VA_ARGS__))

extern "C" int cogdl_b200_gcn_fused_supported(int64_t K, int64_t Fout) { return (K == fg::KDIM && Fout >= 1 && Fout <= 128) ? 1 : 0; }

// The partials are those of the hub-row pre-pass: the SpMM's, or scatter_max's for the max aggregation.
extern "C" int64_t cogdl_b200_gcn_fused_scratch_bytes(int64_t n_chunks, int64_t K) {
  return cogdl_b200_spmm_scratch_bytes(n_chunks, K);
}

extern "C" int64_t cogdl_b200_sage_fused_scratch_bytes(int64_t n_chunks, int64_t K, int32_t aggr) {
  return aggr == COGDL_B200_AGGR_MAX ? cogdl_b200_scatter_max_scratch_bytes(n_chunks, K)
                                     : cogdl_b200_spmm_scratch_bytes(n_chunks, K);
}

extern "C" int cogdl_b200_gcn_fused_f32(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X,
                                        const float *W, const float *bias, const float *rowsum, float *out, float *hub_agg,
                                        int64_t n_rows,
                                        int64_t K, int64_t Fout, int32_t relu, const cogdl_b200_hub_plan_t *plan,
                                        cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_gcn_fused_f32";
  CB_REQUIRE(n_rows >= 0 && K >= 0 && Fout >= 0, "%s: negative size", who);
  if (n_rows == 0 || Fout == 0) return COGDL_B200_OK;
  CB_REQUIRE(cogdl_b200_gcn_fused_supported(K, Fout), "%s: needs K == 128 and 1 <= Fout <= 128 (got K=%lld, Fout=%lld)", who,
             (long long)K, (long long)Fout);
  CB_REQUIRE(rowptr && colind && X && W && out, "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffff00LL, "%s: n_rows must fit int32", who);
  CB_REQUIRE(plan && plan->chunk_edges > 0 && plan->edge_row, "%s: needs a hub plan with edge_row (row-stream form)", who);
  CB_REQUIRE(aligned16(X) && aligned16(W) && aligned16(out), "%s: X, W and out must be 16-byte aligned", who);
  int rc = check_plan(plan, cogdl_b200_gcn_fused_scratch_bytes(plan->n_chunks, K));
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (plan->n_chunks > 0) {
    CB_REQUIRE(hub_agg && aligned16(hub_agg), "%s: hub_agg scratch [n_rows, 128] is required when the plan has hub rows", who);
    rc = spmm_hub_rows_only(rowptr, colind, val, X, hub_agg, K, plan, s);
    if (rc) return rc;
  }
  fg::Params p;
  p.rowptr = rowptr; p.colind = colind; p.val = val; p.edge_row = plan->edge_row; p.X = X; p.W = W; p.bias = bias;
  p.hub_agg = hub_agg ? hub_agg : X; p.rowsum = rowsum; p.out = out; p.n_rows = (int)n_rows; p.Fout = (int)Fout;
  p.Npad = Fout <= fg::WG_N ? fg::WG_N : 2 * fg::WG_N; p.chunk_edges = plan->chunk_edges; p.relu = relu;
  p.n_tiles = (int)ceil_div(n_rows, fg::TILE_M);
  p.row_scale = nullptr; p.S = nullptr;
  FG_NOTE(plan->n_chunks > 0, "cogdl_b200::fg::fused_layer_kernel<gcn, 2 groups x tile 64x%d, K=128, bf16x3 split, wgmma m64n32k16>",
          p.Npad);
  return fg::launch<fg::AGG_SUM, fg::EPI_BIAS>(p, s);
}

extern "C" int cogdl_b200_sage_fused_f32(const int32_t *rowptr, const int32_t *colind, const float *val, const float *row_scale,
                                         const float *X, const float *W_neigh, const float *S, float *out, float *hub_agg,
                                         int64_t n_rows, int64_t K, int64_t Fout, int32_t aggr, int32_t relu,
                                         const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_sage_fused_f32";
  CB_REQUIRE(n_rows >= 0 && K >= 0 && Fout >= 0, "%s: negative size", who);
  CB_REQUIRE(aggr == COGDL_B200_AGGR_SUM || aggr == COGDL_B200_AGGR_MAX, "%s: aggr must be COGDL_B200_AGGR_SUM or _MAX (got %d)",
             who, (int)aggr);
  if (n_rows == 0 || Fout == 0) return COGDL_B200_OK;
  CB_REQUIRE(cogdl_b200_gcn_fused_supported(K, Fout), "%s: needs K == 128 and 1 <= Fout <= 128 (got K=%lld, Fout=%lld)", who,
             (long long)K, (long long)Fout);
  CB_REQUIRE(rowptr && colind && X && W_neigh && S && out, "%s: null pointer", who);
  CB_REQUIRE(aggr == COGDL_B200_AGGR_SUM || (!val && !row_scale), "%s: max aggregation takes no edge values or row scale", who);
  CB_REQUIRE(n_rows < 0x7fffff00LL, "%s: n_rows must fit int32", who);
  CB_REQUIRE(plan && plan->chunk_edges > 0 && plan->edge_row, "%s: needs a hub plan with edge_row (row-stream form)", who);
  CB_REQUIRE(aligned16(X) && aligned16(W_neigh) && aligned16(S) && aligned16(out), "%s: X, W_neigh, S and out must be 16-byte aligned",
             who);
  int rc = check_plan(plan, cogdl_b200_sage_fused_scratch_bytes(plan->n_chunks, K, aggr));
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (plan->n_chunks > 0) {
    CB_REQUIRE(hub_agg && aligned16(hub_agg), "%s: hub_agg scratch [n_rows, 128] is required when the plan has hub rows", who);
    rc = aggr == COGDL_B200_AGGR_MAX ? smax_hub_rows_only(rowptr, colind, X, hub_agg, K, plan, s)
                                     : spmm_hub_rows_only(rowptr, colind, val, X, hub_agg, K, plan, s);
    if (rc) return rc;
  }
  fg::Params p;
  p.rowptr = rowptr; p.colind = colind; p.val = val; p.edge_row = plan->edge_row; p.X = X; p.W = W_neigh; p.bias = nullptr;
  p.hub_agg = hub_agg ? hub_agg : X; p.rowsum = nullptr; p.out = out; p.n_rows = (int)n_rows; p.Fout = (int)Fout;
  p.Npad = Fout <= fg::WG_N ? fg::WG_N : 2 * fg::WG_N; p.chunk_edges = plan->chunk_edges; p.relu = relu;
  p.n_tiles = (int)ceil_div(n_rows, fg::TILE_M);
  p.row_scale = row_scale; p.S = S;
  if (aggr == COGDL_B200_AGGR_MAX) {
    FG_NOTE(plan->n_chunks > 0,
            "cogdl_b200::fg::fused_layer_kernel<sage-max, 2 groups x tile 64x%d, K=128, bf16x3 split, wgmma m64n32k16>", p.Npad);
    return fg::launch<fg::AGG_MAX, fg::EPI_SELF>(p, s);
  }
  FG_NOTE(plan->n_chunks > 0,
          "cogdl_b200::fg::fused_layer_kernel<sage-sum%s, 2 groups x tile 64x%d, K=128, bf16x3 split, wgmma m64n32k16>",
          row_scale ? "+row_scale" : "", p.Npad);
  return fg::launch<fg::AGG_SUM, fg::EPI_SELF>(p, s);
}

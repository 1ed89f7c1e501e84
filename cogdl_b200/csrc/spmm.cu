// spmm.cu -- weighted / unweighted CSR SpMM for sm_90a.
//
//   Y[i,:] = sum_{p in row i} val[p] * X[colind[p],:]
//
// Replaces the reference's GE-SpMM kernels (cogdl/operators/spmm/spmm_kernel.cu:7-512) behind
// spmm.csr_spmm / csr_spmm_no_edge_value (spmm.cpp:22-70).  HBM/L2-bound gather: 4F+8 bytes per
// edge, no reuse => no tensor cores; what matters is coalescing, bytes in flight and balance.
//
// Design (H100):
//   * a GROUP of lanes owns one work item (a row, or one edge chunk of a hub row); each lane
//     owns NV 16-byte vectors of the feature row, so one warp-wide LDG.128 moves a full
//     512-byte row for F = 128 (the reference moves 2 x 128 B with scalar loads and re-reads
//     the indices per 64-column tile);
//   * colind/val are fetched one GROUP-wide coalesced slab at a time with L1::no_allocate and
//     broadcast by shuffle (no shared memory, no block barrier); the next slab is prefetched
//     while the current one is being gathered;
//   * UNROLL independent row gathers are issued before any is consumed (8 x 512 B per warp in
//     flight): with ~32 resident warps/SM that is ~128 KB in flight per SM, above the
//     latency x bandwidth product of HBM3 (~15 KB/SM at 3.35 TB/s over 132 SMs);
//   * rows longer than the hub plan's chunk are cut into chunks that are scheduled first
//     (lowest block indices), partial sums are combined in chunk order by the last chunk to
//     arrive => deterministic; the reference serialises a hub on one warp;
//   * per output element the accumulation is in CSR order with separate fp32 mul and add, so
//     unsplit rows are bit-identical to the reference CPU SpMM (spmm_cpu.cpp:24-36);
//   * 64-bit row offsets (the reference's `int offset = colInd * k` overflows at N*F >= 2^31).
#include "spmm.cuh"

#include <cuda_fp16.h>

#include <cstdlib>

namespace cogdl_b200 {

// ------------------------------------------------------------------------------------------
// fp16 storage, fp32 accumulation.  One lane owns 4 halves (8 bytes); a warp covers 128
// columns per pass.  (Reference: spmm_test{0,1,2}_half accumulate in half, spmm_kernel.cu:
// 222-250,311-368,442-512 -- we keep fp32 accumulators, a documented improvement.)
// ------------------------------------------------------------------------------------------
struct SpmmHalfParams {
  const int *rowptr;
  const int *colind;
  const __half *val;
  const __half *X;
  __half *Y;
  int64_t n_rows;
  int F;
  HubView hub;
};

template <bool HAS_VAL, bool VEC>
__global__ void __launch_bounds__(256) spmm_half_kernel(const SpmmHalfParams p) {
  constexpr int U = 8;
  constexpr int W = VEC ? 4 : 1;  // halves per lane per pass
  const int lane = threadIdx.x & 31;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const WorkItem w = decode_item(tid / 32, p.n_rows, p.rowptr, p.hub);
  float *P = reinterpret_cast<float *>(p.hub.partials);

  for (int tile0 = 0; tile0 < p.F; tile0 += 32 * W) {
    const int col = tile0 + lane * W;
    const bool colok = col < p.F;
    float acc[W];
#pragma unroll
    for (int t = 0; t < W; ++t) acc[t] = 0.f;

    for (int base = w.lb; base < w.hb; base += 32) {
      const int cnt = min(32, w.hb - base);
      int c = 0;
      float v = 0.f;
      if (base + lane < w.hb) {
        c = ld_stream(p.colind + base + lane);
        v = HAS_VAL ? __half2float(p.val[base + lane]) : 1.f;
      }
#pragma unroll 1
      for (int j = 0; j < cnt; j += U) {
        float x[U][W];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, c, j + u);
          if (j + u < cnt && colok) {
            const __half *xp = p.X + (int64_t)cj * p.F + col;
            if constexpr (VEC) {
              const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(xp));
              const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
              const float2 b = __half22float2(*reinterpret_cast<const __half2 *>(&raw.y));
              x[u][0] = a.x; x[u][1] = a.y; x[u][2] = b.x; x[u][3] = b.y;
            } else {
              x[u][0] = __half2float(__ldg(xp));
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float vj = __shfl_sync(FULL, v, j + u);
          if (j + u < cnt && colok) {
#pragma unroll
            for (int t = 0; t < W; ++t) acc[t] = fmaf(vj, x[u][t], acc[t]);
          }
        }
      }
    }
    if (!w.is_chunk) {
      if (w.active && colok) {
        __half *yp = p.Y + (int64_t)w.row * p.F + col;
#pragma unroll
        for (int t = 0; t < W; ++t) yp[t] = __float2half_rn(acc[t]);
      }
    } else if (colok) {
#pragma unroll
      for (int t = 0; t < W; ++t) st_cg(P + (int64_t)w.slot * p.F + col + t, acc[t]);
    }
  }
  if ((tid - lane) / 32 < p.hub.n_chunks) {
    if (hub_arrive_last<32>(w, p.hub, lane)) {
      for (int col = lane; col < p.F; col += 32) {
        float s = 0.f;
        for (int q = 0; q < w.n_row_chunks; ++q) s += ld_cg(P + (int64_t)(w.first + q) * p.F + col);
        p.Y[(int64_t)w.row * p.F + col] = __float2half_rn(s);
      }
    }
  }
}

// Only the hub rows (degree > plan chunk) of Y = A @ X: the hub-chunk items of the row-stream kernel with
// their in-order combine, no segments.  Used by the fused GCN layer (fused_gcn.cu), which aggregates every
// other row straight into shared memory.  F % 4 == 0, 16-byte aligned X / Y.
int spmm_hub_rows_only(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X, float *Y,
                       int64_t F, const cogdl_b200_hub_plan_t *plan, cudaStream_t stream) {
  SpmmParams p;
  p.rowptr = rowptr; p.colind = colind; p.val = val; p.X0 = X; p.X1 = X; p.Y = Y; p.n_rows = 0;
  p.hub = hub_view(plan);
  p.hub.n_segs = 0;
  p.FV = (int)(F / 4);
  if (p.hub.n_chunks == 0) return COGDL_B200_OK;
  const StreamParams q = to_stream(p);
  if (p.FV <= 32) return launch_stream<float4, 1, 4, 5, false>(q, stream);
  return launch_stream<float4, 2, 4, 1>(q, stream);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_spmm_scratch_bytes(int64_t n_chunks, int64_t F) {
  return n_chunks > 0 && F > 0 ? n_chunks * F * (int64_t)sizeof(float) : 0;
}

extern "C" int cogdl_b200_spmm_csr_f32_ex(const int32_t *rowptr, const int32_t *colind, const float *val,
                                          const float *X, int64_t x_rows, float *Y, int64_t n_rows, int64_t F,
                                          int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                          cogdl_b200_stream_t stream) {
  return spmm_entry<EPI_NONE>(rowptr, colind, val, X, INT64_MAX, nullptr, Y, n_rows, F, plan, stream,
                           "cogdl_b200_spmm_csr_f32_ex", nullptr, 0, 0, x_rows, panels);
}

extern "C" int cogdl_b200_spmm_csr_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                                       const float *X, float *Y, int64_t n_rows, int64_t F,
                                       const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return cogdl_b200_spmm_csr_f32_ex(rowptr, colind, val, X, n_rows, Y, n_rows, F, 0, plan, stream);
}

extern "C" int cogdl_b200_spmm_csr_f32_2src(const int32_t *rowptr, const int32_t *colind, const float *val,
                                            const float *X0, int64_t n0, const float *X1, float *Y,
                                            int64_t n_rows, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                            cogdl_b200_stream_t stream) {
  CB_REQUIRE(n0 >= 0, "cogdl_b200_spmm_csr_f32_2src: n0 < 0");
  CB_REQUIRE(X1 != nullptr || n0 == INT64_MAX, "cogdl_b200_spmm_csr_f32_2src: X1 is null");
  return spmm_entry<EPI_NONE>(rowptr, colind, val, X0, n0, X1, Y, n_rows, F, plan, stream,
                           "cogdl_b200_spmm_csr_f32_2src");
}

extern "C" int cogdl_b200_spmm_csr_f16(const int32_t *rowptr, const int32_t *colind, const void *val,
                                       const void *X, void *Y, int64_t n_rows, int64_t F,
                                       const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && F >= 0, "cogdl_b200_spmm_csr_f16: negative size");
  if (n_rows == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && X && Y, "cogdl_b200_spmm_csr_f16: null pointer");
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "cogdl_b200_spmm_csr_f16: sizes must fit int32");
  int rc = check_plan(plan, cogdl_b200_spmm_scratch_bytes(plan ? plan->n_chunks : 0, F));
  if (rc) return rc;
  SpmmHalfParams p;
  p.rowptr = rowptr; p.colind = colind; p.val = (const __half *)val; p.X = (const __half *)X;
  p.Y = (__half *)Y; p.n_rows = n_rows; p.F = (int)F; p.hub = hub_view(plan);
  const bool vec = (F % 4 == 0) && ((reinterpret_cast<uintptr_t>(X) & 7u) == 0);
  const int64_t items = (int64_t)p.hub.n_chunks + n_rows;
  const int64_t blocks = ceil_div(items * 32, 256);
  CB_REQUIRE(blocks <= 0x7fffffffLL, "cogdl_b200_spmm_csr_f16: problem too large");
  dim3 grid((unsigned)blocks);
  cudaStream_t s = (cudaStream_t)stream;
  note_kernel("cogdl_b200::spmm_half_kernel<%s,%s>", val ? "weighted" : "unweighted", vec ? "vec" : "scalar");
  if (vec) {
    if (val) spmm_half_kernel<true, true><<<grid, 256, 0, s>>>(p);
    else spmm_half_kernel<false, true><<<grid, 256, 0, s>>>(p);
  } else {
    if (val) spmm_half_kernel<true, false><<<grid, 256, 0, s>>>(p);
    else spmm_half_kernel<false, false><<<grid, 256, 0, s>>>(p);
  }
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_spmm_csr_f32_peers(const int32_t *rowptr, const int32_t *colind, const float *val,
                                             const float *X_local, int64_t n_local, const float *const *peer_ptrs,
                                             int32_t n_peers, int32_t owner_shift, float *Y, int64_t n_rows,
                                             int64_t F, const cogdl_b200_hub_plan_t *plan,
                                             cogdl_b200_stream_t stream) {
  CB_REQUIRE(peer_ptrs && n_peers >= 1 && n_peers <= 8, "cogdl_b200_spmm_csr_f32_peers: need 1..8 peer pointers");
  CB_REQUIRE(owner_shift >= 1 && owner_shift <= 28 && n_local >= 0, "cogdl_b200_spmm_csr_f32_peers: bad owner_shift / n_local");
  for (int i = 0; i < n_peers; ++i) CB_REQUIRE(peer_ptrs[i], "cogdl_b200_spmm_csr_f32_peers: null peer pointer %d", i);
  return spmm_entry<EPI_NONE>(rowptr, colind, val, X_local, n_local, nullptr, Y, n_rows, F, plan, stream,
                           "cogdl_b200_spmm_csr_f32_peers", peer_ptrs, n_peers, owner_shift);
}

// scatter_max.cu -- neighbour max with argmax (GraphSAGE max aggregator) for sm_90a.
//
//   out[i,f]    = max_{p in row i} X[colind[p], f]
//   argmax[i,f] = colind of the FIRST edge (CSR order) attaining the max   (strict `<` update)
//
// Replaces scatter_max_forward / scatter_max_backward (cogdl/operators/scatter_max/
// scatter_max.cu:5-42; one block per row, F scalar threads, every thread re-reads colind).
// Same gather skeleton as the SpMM (lane-owned 16-byte vectors, index slab broadcast by shuffle,
// UNROLL gathers in flight, hub rows cut into chunks).  Max/argmax with a first-wins tie rule is
// order-preserving under in-order combination of chunk partials, so the result is bit-exact
// with and without a hub plan.
//
// Fixed semantics (documented divergences, see include/cogdl_b200.h): running max starts at
// -inf (reference: FLT_MIN); degree-0 rows -> out 0, argmax -1 (reference: uninitialised);
// backward zero-fills its output (reference: torch::empty, never zeroed).
#include "common.cuh"

#include <math_constants.h>

#include <cstdlib>

namespace cogdl_b200 {

struct SmaxParams {
  const int *rowptr;
  const int *colind;
  const float *X;
  float *out;
  int *argmax;
  int64_t n_rows;
  int FV;
  HubView hub;
};

template <typename VecT> struct IdxOf;
template <> struct IdxOf<float4> { using type = int4; };
template <> struct IdxOf<float> { using type = int; };

__device__ __forceinline__ void upd(float &m, int &id, float x, int c) {
  if (m < x) { m = x; id = c; }
}
__device__ __forceinline__ void upd(float4 &m, int4 &id, const float4 &x, int c) {
  upd(m.x, id.x, x.x, c); upd(m.y, id.y, x.y, c); upd(m.z, id.z, x.z, c); upd(m.w, id.w, x.w, c);
}
__device__ __forceinline__ void upd2(float &m, int &id, float x, int c) { upd(m, id, x, c); }
__device__ __forceinline__ void upd2(float4 &m, int4 &id, const float4 &x, const int4 &c) {
  upd(m.x, id.x, x.x, c.x); upd(m.y, id.y, x.y, c.y); upd(m.z, id.z, x.z, c.z); upd(m.w, id.w, x.w, c.w);
}
__device__ __forceinline__ void init_acc(float &m, int &id) { m = -CUDART_INF_F; id = -1; }
__device__ __forceinline__ void init_acc(float4 &m, int4 &id) {
  m = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
  id = make_int4(-1, -1, -1, -1);
}
__device__ __forceinline__ void zero_acc(float &m) { m = 0.f; }
__device__ __forceinline__ void zero_acc(float4 &m) { m = make_float4(0.f, 0.f, 0.f, 0.f); }
// (max, argmax) partial of one lane vector, as the last chunk of a hub row combines them
template <typename VecT>
struct MaxAcc {
  VecT m;
  typename IdxOf<VecT>::type id;
};
__device__ __forceinline__ int4 ld_cg(const int4 *p) { return __ldcg(p); }
__device__ __forceinline__ void st_cg(int4 *p, int4 v) { __stcg(p, v); }
__device__ __forceinline__ void st_stream(int4 *p, int4 v) { __stcs(p, v); }

template <typename VecT, int GROUP, int NV>
__global__ void __launch_bounds__(256) scatter_max_fwd_kernel(const SmaxParams p) {
  using IdxT = typename IdxOf<VecT>::type;
  constexpr int U0 = (NV == 1) ? 8 : 4;
  constexpr int U = U0 < GROUP ? U0 : GROUP;
  constexpr int TILE = GROUP * NV;
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const WorkItem w = decode_item(tid / GROUP, p.n_rows, p.rowptr, p.hub);
  const bool warp_has_chunk = (tid - lane) / GROUP < p.hub.n_chunks;

  const VecT *X = reinterpret_cast<const VecT *>(p.X);
  VecT *O = reinterpret_cast<VecT *>(p.out);
  IdxT *A = reinterpret_cast<IdxT *>(p.argmax);
  // partial scratch: [n_chunks, F] values followed by [n_chunks, F] argmax ids
  VecT *PV = reinterpret_cast<VecT *>(p.hub.partials);
  IdxT *PI = reinterpret_cast<IdxT *>(PV + (int64_t)p.hub.n_chunks * p.FV);

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);

  for (int tile0 = 0; tile0 < p.FV; tile0 += TILE) {
    const int cv = tile0 + gl;
    bool colok[NV];
    VecT acc[NV];
    IdxT id[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      colok[k] = (cv + k * GROUP) < p.FV;
      init_acc(acc[k], id[k]);
    }
    int c = 0;
    if (w.lb + gl < w.hb) c = ld_stream(p.colind + w.lb + gl);
    for (int off = 0; off < maxdeg; off += GROUP) {
      const int cnt = min(GROUP, w.hb - w.lb - off);
      int cn = 0;
      if (w.lb + off + GROUP + gl < w.hb) cn = ld_stream(p.colind + w.lb + off + GROUP + gl);
#pragma unroll 1
      for (int j = 0; j < GROUP; j += U) {
        if (GROUP == 32) {
          if (j >= cnt) break;
        } else {
          if (!__any_sync(FULL, j < cnt)) break;
        }
        VecT x[U][NV];
        int cj[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          cj[u] = __shfl_sync(FULL, c, j + u, GROUP);
          if (j + u < cnt) {
            const VecT *xp = X + (int64_t)cj[u] * p.FV + cv;
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) x[u][k] = ld_gather(xp + k * GROUP);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (j + u < cnt) {
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) upd(acc[k], id[k], x[u][k], cj[u]);
          }
        }
      }
      c = cn;
    }
    if (!w.is_chunk) {
      if (w.active) {
        if (w.hb == w.lb) {
#pragma unroll
          for (int k = 0; k < NV; ++k) zero_acc(acc[k]);  // degree-0 row: out = 0, argmax = -1
        }
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (colok[k]) {
            st_stream(O + (int64_t)w.row * p.FV + cv + k * GROUP, acc[k]);
            st_stream(A + (int64_t)w.row * p.FV + cv + k * GROUP, id[k]);
          }
      }
    } else {
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (colok[k]) {
          st_cg(PV + (int64_t)w.slot * p.FV + cv + k * GROUP, acc[k]);
          st_cg(PI + (int64_t)w.slot * p.FV + cv + k * GROUP, id[k]);
        }
    }
  }
  if (warp_has_chunk) {
    if (hub_arrive_last<GROUP>(w, p.hub, gl)) {
      for (int cv = gl; cv < p.FV; cv += GROUP) {
        // chunk order + strict `<` keeps "first max wins"
        const MaxAcc<VecT> m = merge_chunks<1>(
            w.n_row_chunks,
            [&](int q) {
              const int64_t i = (int64_t)(w.first + q) * p.FV + cv;
              return MaxAcc<VecT>{ld_cg(PV + i), ld_cg(PI + i)};
            },
            [](MaxAcc<VecT> &s, const MaxAcc<VecT> &t) { upd2(s.m, s.id, t.m, t.id); });
        st_stream(O + (int64_t)w.row * p.FV + cv, m.m);
        st_stream(A + (int64_t)w.row * p.FV + cv, m.id);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Row-stream form (same skeleton as stream.cuh, with (max, argmax) accumulators): used when the plan
// carries segments and a full warp owns the row (F >= 68 on the float4 path).  Hub chunks write
// (value, argmax) partials that the last chunk to arrive combines in chunk order with the strict
// `<` rule, so "first max wins" holds across chunks as well: results stay bit-exact.
// ARGMAX == false tracks values only (hub-only pre-pass of the fused SAGE layer): no argmax output and no id
// partials; the values are the same, since the in-order strict `<` combine of the partial maxima is the row's max.
// ------------------------------------------------------------------------------------------
template <int NV, int U, bool ARGMAX = true>
__global__ void __launch_bounds__(256) scatter_max_stream_kernel(const SmaxParams p) {
  constexpr int TILE = 32 * NV;
  const int lane = threadIdx.x & 31;
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const float4 *X = reinterpret_cast<const float4 *>(p.X);
  float4 *O = reinterpret_cast<float4 *>(p.out);
  int4 *A = reinterpret_cast<int4 *>(p.argmax);
  float4 *PV = reinterpret_cast<float4 *>(p.hub.partials);
  int4 *PI = reinterpret_cast<int4 *>(PV + (int64_t)p.hub.n_chunks * p.FV);

  WorkItem w;
  int e_begin, e_end, r_begin = 0, r_end = 0;
  const bool is_chunk = item < p.hub.n_chunks;
  if (is_chunk) {
    w = decode_item(item, 0, p.rowptr, p.hub);
    e_begin = w.lb; e_end = w.hb;
  } else {
    const int64_t seg = item - p.hub.n_chunks;
    if (seg >= p.hub.n_segs) return;
    const int2 rr = __ldg(p.hub.segs + seg);
    r_begin = rr.x; r_end = rr.y;
    e_begin = __ldg(p.rowptr + rr.x); e_end = __ldg(p.rowptr + rr.y);
  }

  for (int tile0 = 0; tile0 < p.FV; tile0 += TILE) {
    const int cv = tile0 + lane;
    bool colok[NV];
    float4 acc[NV];
    int4 id[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) { colok[k] = (cv + k * 32) < p.FV; init_acc(acc[k], id[k]); }
    if (!is_chunk && p.hub.n_empty_rows > 0) {   // degree-0 rows: out = 0, argmax = -1
      for (int rb = r_begin; rb < r_end; rb += 32) {
        const int row = rb + lane;
        unsigned m = __ballot_sync(FULL, row < r_end && __ldg(p.rowptr + row + 1) == __ldg(p.rowptr + row));
        while (m) {
          const int k0 = __ffs(m) - 1;
          m &= m - 1;
#pragma unroll
          for (int k = 0; k < NV; ++k)
            if (colok[k]) {
              st_stream(O + (int64_t)(rb + k0) * p.FV + cv + k * 32, make_float4(0.f, 0.f, 0.f, 0.f));
              if (ARGMAX) st_stream(A + (int64_t)(rb + k0) * p.FV + cv + k * 32, make_int4(-1, -1, -1, -1));
            }
        }
      }
    }
    for (int e = e_begin; e < e_end; e += 32) {
      const int cnt = min(32, e_end - e);
      int c = 0, rid = -1, rnx = -1;
      if (lane < cnt) {
        c = ld_stream(p.colind + e + lane);
        if (!is_chunk) {
          rid = ld_stream(p.hub.edge_row + e + lane);
          if (e + lane + 1 < e_end) rnx = __ldg(p.hub.edge_row + e + lane + 1);
        }
      }
      const unsigned endmask = is_chunk ? 0u : __ballot_sync(FULL, lane < cnt && rid != rnx);
#pragma unroll 1
      for (int j = 0; j < cnt; j += U) {
        const unsigned em = endmask >> j;
        float4 x[U][NV];
        int cj[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          cj[u] = __shfl_sync(FULL, c, j + u);
          if (j + u < cnt) {
            const float4 *xp = X + (int64_t)cj[u] * p.FV + cv;
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) x[u][k] = ld_gather(xp + k * 32);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (j + u < cnt) {
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) upd(acc[k], id[k], x[u][k], cj[u]);
            if ((em >> u) & 1u) {   // last edge of its row (warp-uniform)
              const int rj = __shfl_sync(FULL, rid, j + u);
#pragma unroll
              for (int k = 0; k < NV; ++k)
                if (colok[k]) {
                  st_stream(O + (int64_t)rj * p.FV + cv + k * 32, acc[k]);
                  if (ARGMAX) st_stream(A + (int64_t)rj * p.FV + cv + k * 32, id[k]);
                  init_acc(acc[k], id[k]);
                }
            }
          }
        }
      }
    }
    if (is_chunk) {
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (colok[k]) {
          st_cg(PV + (int64_t)w.slot * p.FV + cv + k * 32, acc[k]);
          if (ARGMAX) st_cg(PI + (int64_t)w.slot * p.FV + cv + k * 32, id[k]);
        }
    }
  }
  if (is_chunk) {
    if (hub_arrive_last<32>(w, p.hub, lane)) {
      for (int cv = lane; cv < p.FV; cv += 32) {
        const MaxAcc<float4> m = merge_chunks<1>(
            w.n_row_chunks,
            [&](int q) {
              const int64_t i = (int64_t)(w.first + q) * p.FV + cv;
              return MaxAcc<float4>{ld_cg(PV + i), ARGMAX ? ld_cg(PI + i) : make_int4(-1, -1, -1, -1)};
            },
            [](MaxAcc<float4> &s, const MaxAcc<float4> &t) { upd2(s.m, s.id, t.m, t.id); });
        st_stream(O + (int64_t)w.row * p.FV + cv, m.m);
        if (ARGMAX) st_stream(A + (int64_t)w.row * p.FV + cv, m.id);
      }
    }
  }
}

// Row-stream form whenever the plan has segments and a row is wider than 16 vectors: bit-exact either way; products
// shape F=256: 11.38 ms (row-stream form) vs 11.52 ms (row per warp)
template <int NV>
static int launch_smax_stream(const SmaxParams &p, cudaStream_t stream) {
  constexpr int U = NV == 1 ? 4 : 2;
  return launch_items(scatter_max_stream_kernel<NV, U>, p, (int64_t)p.hub.n_chunks + p.hub.n_segs, 32, stream,
                      "scatter_max", "cogdl_b200::scatter_max_stream_kernel<NV=%d,U=%d>", NV, U);
}

template <typename VecT, int GROUP, int NV>
static int launch_smax(const SmaxParams &p, cudaStream_t stream) {
  return launch_items(scatter_max_fwd_kernel<VecT, GROUP, NV>, p, (int64_t)p.hub.n_chunks + p.n_rows, GROUP, stream,
                      "scatter_max", "cogdl_b200::scatter_max_fwd_kernel<%s,GROUP=%d,NV=%d>",
                      sizeof(VecT) == 16 ? "float4" : "float", GROUP, NV);
}

template <typename VecT>
static int dispatch_smax(const SmaxParams &p, cudaStream_t s) {
  const int fv = p.FV;
  if constexpr (sizeof(VecT) == 16) {
    if (fv > 16 && p.hub.n_segs > 0)
      return fv <= 32 ? launch_smax_stream<1>(p, s) : launch_smax_stream<2>(p, s);
  }
  if (fv <= 1) return launch_smax<VecT, 1, 1>(p, s);
  if (fv <= 2) return launch_smax<VecT, 2, 1>(p, s);
  if (fv <= 4) return launch_smax<VecT, 4, 1>(p, s);
  if (fv <= 8) return launch_smax<VecT, 8, 1>(p, s);
  if (fv <= 16) return launch_smax<VecT, 16, 1>(p, s);
  if (fv <= 32) return launch_smax<VecT, 32, 1>(p, s);
  return launch_smax<VecT, 32, 2>(p, s);
}

// Only the hub rows (degree > plan chunk) of the max values, no argmax: the hub-chunk items of the row-stream
// kernel with their in-order combine, no segments.  Used by the fused
// SAGE layer (fused_gcn.cu), which aggregates every other row straight into shared memory.  F == 128, 16-byte
// aligned X / Y; plan->partials cogdl_b200_scatter_max_scratch_bytes(n_chunks, F) bytes.
int smax_hub_rows_only(const int32_t *rowptr, const int32_t *colind, const float *X, float *Y, int64_t F,
                       const cogdl_b200_hub_plan_t *plan, cudaStream_t stream) {
  SmaxParams p;
  p.rowptr = rowptr; p.colind = colind; p.X = X; p.out = Y; p.argmax = nullptr; p.n_rows = 0;
  p.hub = hub_view(plan);
  p.hub.n_segs = 0;
  p.FV = (int)(F / 4);
  if (p.hub.n_chunks == 0) return COGDL_B200_OK;
  if (p.FV != 32) return set_error(COGDL_B200_EINVAL, "smax_hub_rows_only: F must be 128");
  const int64_t blocks = ceil_div((int64_t)p.hub.n_chunks * 32, 256);
  note_kernel("cogdl_b200::scatter_max_stream_kernel<NV=1,U=4,values_only>");
  scatter_max_stream_kernel<1, 4, false><<<(unsigned)blocks, 256, 0, stream>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

// gx[argmax[i,f], f] += g[i,f]  (red.global.add.f32; gx zero-filled by the caller below)
__global__ void __launch_bounds__(256) scatter_max_bwd_kernel(const float *__restrict__ g,
                                                              const int *__restrict__ argmax,
                                                              float *__restrict__ gx, int64_t total, int F) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int id = ld_stream(argmax + t);
    if (id >= 0) atomicAdd(gx + (int64_t)id * F + (t % F), ld_stream(g + t));
  }
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

// (value, argmax) per chunk and column
extern "C" int64_t cogdl_b200_scatter_max_scratch_bytes(int64_t n_chunks, int64_t F) {
  return n_chunks > 0 && F > 0 ? n_chunks * F * 8 : 0;
}

extern "C" int cogdl_b200_scatter_max_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *X,
                                              float *out, int32_t *argmax, int64_t n_rows, int64_t F,
                                              const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && F >= 0, "cogdl_b200_scatter_max_fwd_f32: negative size");
  if (n_rows == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && X && out && argmax, "cogdl_b200_scatter_max_fwd_f32: null pointer");
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "cogdl_b200_scatter_max_fwd_f32: sizes must fit int32");
  int rc = check_plan(plan, cogdl_b200_scatter_max_scratch_bytes(plan ? plan->n_chunks : 0, F));
  if (rc) return rc;
  SmaxParams p;
  p.rowptr = rowptr; p.colind = colind; p.X = X; p.out = out; p.argmax = argmax; p.n_rows = n_rows;
  p.hub = hub_view(plan);
  const bool vec = (F % 4 == 0) && aligned16(X) && aligned16(out) && aligned16(argmax) &&
                   (p.hub.n_chunks == 0 || aligned16(p.hub.partials));
  if (vec) {
    p.FV = (int)(F / 4);
    return dispatch_smax<float4>(p, (cudaStream_t)stream);
  }
  p.FV = (int)F;
  return dispatch_smax<float>(p, (cudaStream_t)stream);
}

extern "C" int cogdl_b200_scatter_max_bwd_f32(const float *g, const int32_t *argmax, float *gx,
                                              int64_t n_rows, int64_t n_src, int64_t F,
                                              cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && n_src >= 0 && F >= 0, "cogdl_b200_scatter_max_bwd_f32: negative size");
  if (n_src == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(gx, "cogdl_b200_scatter_max_bwd_f32: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  CB_CUDA(cudaMemsetAsync(gx, 0, (size_t)(n_src * F) * sizeof(float), s));
  if (n_rows == 0) return COGDL_B200_OK;
  CB_REQUIRE(g && argmax, "cogdl_b200_scatter_max_bwd_f32: null pointer");
  CB_REQUIRE(F < 0x7fffffffLL, "cogdl_b200_scatter_max_bwd_f32: F must fit int32");
  const int64_t total = n_rows * F;
  int64_t blocks = ceil_div(total, 256);
  if (blocks > NUM_SMS * 32) blocks = NUM_SMS * 32;
  note_kernel("cogdl_b200::scatter_max_bwd_kernel");
  scatter_max_bwd_kernel<<<(unsigned)blocks, 256, 0, s>>>(g, argmax, gx, total, (int)F);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

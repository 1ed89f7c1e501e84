// rgcn.cu -- R-GCN relational aggregation under a basis decomposition, sm_90a.
//
// With W_t = sum_b coef[t,b] V_b, the layer's relational sum sum_t A_t x W_t is agg.view(N, B*F) @ V.view(B*F, F_out)
// with the fan-out aggregation
//
//   Y[i,b,:] = sum_{q in row i} fl(w[q] * coef[type[q], b]) * X[colind[q], :]          b = 0 .. B-1
//
// (cogdl/layers/rgcn_layer.py:118-150 forms x @ W_t for every relation instead: a [T, N, F_out] tensor).  Each edge
// reads its column, weight and type once and gathers its X row once; the row then feeds B accumulators.  Per output
// element the accumulation is in CSR order with a separate fp32 multiply and add from 0, and hub rows are cut into the
// plan's chunks and merged in chunk order -- the plain SpMM's order and rounding -- so Y[:, b, :] is bit-identical to
// the SpMM of X with per-slot values fl(w * coef[type, b]) on the same structure, and reproducible run to run.
//
// Work items are the row-stream items of the hub plan (stream.cuh): hub chunks first, then segments of consecutive
// non-hub rows, one warp each.  A warp walks its rows one after the other; a row's slots are loaded 32 at a time (one
// coalesced load each for column, weight and type), each lane forms the coefficients of its own slot, and the gathers
// go U at a time with the column and the coefficients broadcast by shuffles.  Lanes own 32 vectors (float4 when F % 4
// == 0 and the buffers are aligned, else floats) of the row and BT bases; wider rows loop over column tiles and larger
// B over basis tiles (DESIGN 3.17).
//
// PER_BASIS: X is [x_rows, B, F] and basis b gathers X[colind[q], b, :] -- the standalone aggregation's feature
// gradient, sum_b A_b^T dY[:, b, :], before its sum over b.
//
// The edge dot for d coef: P[q, b] = fl(w[q] * <G[row_q, b, :], X[colind[q], :]>) in slot order, one warp per item
// of the same plan; reduced per type by the caller (an unweighted SpMM over the type-grouped slot index).
#include "common.cuh"
#include "stream.cuh"

namespace cogdl_b200 {

// Bases per pass: 8 accumulators of float4 are 32 registers per lane, no spills at U = 4 (ptxas -v, DESIGN 3.17);
// LinkPredictRGCN's default num_bases = 5 runs in one pass.
constexpr int RGCN_BT = 8;
constexpr int RGCN_U = 4;

struct RgcnParams {
  const int *rowptr;
  const int *colind;
  const int *etype;
  const float *w;
  const float *coef;   // [T, B]
  int B;
  const float *X;      // [x_rows, F] (or [x_rows, B, F] with PER_BASIS)
  float *Y;            // [n_rows, B, F]
  const float *G;      // edge dot: [n_rows, B, F]
  float *P;            // edge dot: [nnz, B]
  int ldv;             // F in VecT units
  HubView hub;
};

// Rows [r0, r1) of a segment, or the edge range of one hub chunk, as one warp's work.
struct RgcnItem {
  bool chunk;
  WorkItem w;
  int r0, r1;
};

__device__ __forceinline__ bool rgcn_item(const RgcnParams &p, int64_t item, RgcnItem &it) {
  it.chunk = item < p.hub.n_chunks;
  if (it.chunk) {
    it.w = decode_item(item, 0, p.rowptr, p.hub);
    it.r0 = it.w.row; it.r1 = it.w.row + 1;
    return true;
  }
  const int64_t seg = item - p.hub.n_chunks;
  if (seg >= p.hub.n_segs) return false;
  const int2 rr = __ldg(p.hub.segs + seg);
  it.r0 = rr.x; it.r1 = rr.y;
  return true;
}

// Accumulate the slots [e, e_end) into acc[0 .. nb) for bases b0 .. b0 + nb of the column vector cv.
template <typename VecT, bool PER_BASIS>
__device__ __forceinline__ void fanout_range(const RgcnParams &p, int e, const int e_end, const int b0, const int nb,
                                             const int cv, const bool colok, const int lane, VecT (&acc)[RGCN_BT]) {
  const VecT *X = reinterpret_cast<const VecT *>(p.X) + cv;
  const int64_t xrow = PER_BASIS ? (int64_t)p.B * p.ldv : p.ldv;
  constexpr int U = PER_BASIS ? 1 : RGCN_U;         // PER_BASIS gathers nb vectors per slot: one slot at a time
  for (; e < e_end; e += 32) {
    const int cnt = min(32, e_end - e);
    const int q = e + lane;
    int c = 0;
    float cf[RGCN_BT];
#pragma unroll
    for (int k = 0; k < RGCN_BT; ++k) cf[k] = 0.f;
    if (q < e_end) {
      c = ld_stream(p.colind + q);
      const float wq = ld_stream(p.w + q);
      const float *cr = p.coef + (int64_t)ld_stream(p.etype + q) * p.B + b0;
#pragma unroll
      for (int k = 0; k < RGCN_BT; ++k)
        if (k < nb) cf[k] = __fmul_rn(wq, __ldg(cr + k));
    }
#pragma unroll 1
    for (int j = 0; j < cnt; j += U) {
      const bool full = j + U <= cnt;
      VecT x[U][PER_BASIS ? RGCN_BT : 1];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int cj = __shfl_sync(FULL, c, j + u);
        if ((full || j + u < cnt) && colok) {
          const VecT *xp = X + (int64_t)cj * xrow;
          if constexpr (PER_BASIS) {
#pragma unroll
            for (int k = 0; k < RGCN_BT; ++k)
              if (k < nb) x[u][k] = ld_gather(xp + (int64_t)(b0 + k) * p.ldv);
          } else {
            x[u][0] = ld_gather(xp);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (full || j + u < cnt) {
#pragma unroll
          for (int k = 0; k < RGCN_BT; ++k) {
            const float ck = __shfl_sync(FULL, cf[k], j + u);
            if (k < nb && colok) axpy_rn(acc[k], ck, x[u][PER_BASIS ? k : 0]);
          }
        }
      }
    }
  }
}

template <typename VecT, bool PER_BASIS>
__global__ void __launch_bounds__(STREAM_BLOCK, 1) rgcn_fanout_kernel(const RgcnParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  RgcnItem it;
  if (!rgcn_item(p, item, it)) return;
  VecT *Y = reinterpret_cast<VecT *>(p.Y);
  VecT *Pt = reinterpret_cast<VecT *>(p.hub.partials);
  const int64_t ystride = (int64_t)p.B * p.ldv;   // one output row: B vectors of ldv
  for (int b0 = 0; b0 < p.B; b0 += RGCN_BT) {
    const int nb = min(RGCN_BT, p.B - b0);
    for (int tile0 = 0; tile0 < p.ldv; tile0 += 32) {
      const int cv = tile0 + lane;
      const bool colok = cv < p.ldv;
      for (int r = it.r0; r < it.r1; ++r) {
        VecT acc[RGCN_BT];
#pragma unroll
        for (int k = 0; k < RGCN_BT; ++k) acc[k] = vzero<VecT>();
        const int lb = it.chunk ? it.w.lb : __ldg(p.rowptr + r), hb = it.chunk ? it.w.hb : __ldg(p.rowptr + r + 1);
        fanout_range<VecT, PER_BASIS>(p, lb, hb, b0, nb, cv, colok, lane, acc);
        VecT *dst = it.chunk ? Pt + (int64_t)it.w.slot * ystride : Y + (int64_t)r * ystride;
#pragma unroll
        for (int k = 0; k < RGCN_BT; ++k) {
          if (k < nb && colok) {
            VecT *yp = dst + (int64_t)(b0 + k) * p.ldv + cv;
            if (it.chunk) st_cg(yp, acc[k]);
            else st_stream(yp, acc[k]);
          }
        }
      }
    }
  }
  if (!it.chunk) return;
  // every basis and column of this chunk's partial is stored: the row's last chunk folds them in chunk order
  if (hub_arrive_last<32>(it.w, p.hub, lane)) {
    for (int b = 0; b < p.B; ++b) {
      for (int cv = lane; cv < p.ldv; cv += 32) {
        const VecT *pp = Pt + (int64_t)it.w.first * ystride + (int64_t)b * p.ldv + cv;
        const VecT s = merge_chunks<8>(it.w.n_row_chunks, [&](int q) { return ld_cg(pp + (int64_t)q * ystride); },
                                       [](VecT &a, const VecT &t) { add_rn(a, t); });
        st_stream(Y + (int64_t)it.w.row * ystride + (int64_t)b * p.ldv + cv, s);
      }
    }
  }
}

__device__ __forceinline__ float dot_rn(const float4 &a, const float4 &b, float s) {
  s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s);
  return fmaf(a.w, b.w, s);
}
__device__ __forceinline__ float dot_rn(const float &a, const float &b, float s) { return fmaf(a, b, s); }

// P[q, b] = fl(w[q] * <G[row_q, b, :], X[colind[q], :]>) for every slot of the item's rows.  Each lane sums its
// columns of every basis of the tile (G's row comes from the L1 after the row's first slot), then a butterfly gives
// every lane the B sums and lane k stores basis k.  Fixed order: reproducible run to run.
template <typename VecT>
__global__ void __launch_bounds__(STREAM_BLOCK, 1) rgcn_edge_dot_kernel(const RgcnParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  RgcnItem it;
  if (!rgcn_item(p, item, it)) return;
  const VecT *G = reinterpret_cast<const VecT *>(p.G);
  const VecT *X = reinterpret_cast<const VecT *>(p.X);
  const int64_t gstride = (int64_t)p.B * p.ldv;
  for (int r = it.r0; r < it.r1; ++r) {
    const int lb = it.chunk ? it.w.lb : __ldg(p.rowptr + r), hb = it.chunk ? it.w.hb : __ldg(p.rowptr + r + 1);
    const VecT *g = G + (int64_t)r * gstride;
    for (int e = lb; e < hb; e += 32) {
      const int cnt = min(32, hb - e);
      int c = 0;
      float wq = 0.f;
      if (e + lane < hb) { c = ld_stream(p.colind + e + lane); wq = ld_stream(p.w + e + lane); }
#pragma unroll 1
      for (int j = 0; j < cnt; ++j) {
        const int cj = __shfl_sync(FULL, c, j);
        const float wj = __shfl_sync(FULL, wq, j);
        const VecT *xp = X + (int64_t)cj * p.ldv;
        for (int b0 = 0; b0 < p.B; b0 += RGCN_BT) {
          const int nb = min(RGCN_BT, p.B - b0);
          float s[RGCN_BT];
#pragma unroll
          for (int k = 0; k < RGCN_BT; ++k) s[k] = 0.f;
          for (int cv = lane; cv < p.ldv; cv += 32) {
            const VecT xv = ld_gather(xp + cv);
#pragma unroll
            for (int k = 0; k < RGCN_BT; ++k)
              if (k < nb) s[k] = dot_rn(__ldg(g + (int64_t)(b0 + k) * p.ldv + cv), xv, s[k]);
          }
          float mine = 0.f;
#pragma unroll
          for (int k = 0; k < RGCN_BT; ++k) {
            if (k < nb) {
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(FULL, s[k], o);
              if (lane == k) mine = s[k];
            }
          }
          if (lane < nb) st_stream(p.P + (int64_t)(e + j) * p.B + b0 + lane, __fmul_rn(wj, mine));
        }
      }
    }
  }
}

template <typename K>
static int launch_rgcn(K kernel, const RgcnParams &p, cudaStream_t stream, const char *who, const char *name,
                       const char *vec) {
  const int64_t warps = (int64_t)p.hub.n_chunks + p.hub.n_segs;
  const int64_t blocks = ceil_div(warps * 32, STREAM_BLOCK);
  if (blocks == 0) return COGDL_B200_OK;
  if (blocks > 0x7fffffffLL) return set_error(COGDL_B200_EINVAL, "%s: problem too large for one launch", who);
  note_kernel("cogdl_b200::%s<%s> block=%d", name, vec, STREAM_BLOCK);
  kernel<<<(unsigned)blocks, STREAM_BLOCK, 0, stream>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

// The checks both entries share; fills p's structure, plan and sizes.
static int rgcn_setup(const char *who, RgcnParams &p, const int32_t *rowptr, const int32_t *colind, const float *w,
                      int64_t n_rows, int64_t B, int64_t F, const cogdl_b200_hub_plan_t *plan) {
  CB_REQUIRE(F > 0 && F < 0x7fffffffLL, "%s: F must be in [1, 2^31), got %lld", who, (long long)F);
  CB_REQUIRE(B > 0 && B <= 4096, "%s: B must be in [1, 4096], got %lld", who, (long long)B);
  CB_REQUIRE(n_rows >= 0 && n_rows < 0x7fffffffLL, "%s: bad row count", who);
  CB_REQUIRE(rowptr && colind && w, "%s: null pointer", who);
  CB_REQUIRE(plan && plan->chunk_edges > 0, "%s: needs a hub plan", who);
  CB_REQUIRE(plan->n_hub_rows <= n_rows && (plan->n_segs > 0 || plan->n_hub_rows == n_rows),
             "%s: the plan does not match the structure's %lld rows (%d hub rows, %d segments)", who,
             (long long)n_rows, plan->n_hub_rows, plan->n_segs);
  p.rowptr = rowptr; p.colind = colind; p.w = w; p.B = (int)B;
  p.hub = hub_view(plan);
  return COGDL_B200_OK;
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_rgcn_aggr_scratch_bytes(int64_t n_chunks, int64_t B, int64_t F) {
  return n_chunks > 0 && B > 0 && F > 0 ? n_chunks * B * F * (int64_t)sizeof(float) : 0;
}

extern "C" int cogdl_b200_rgcn_aggr_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *etype,
                                        const float *w, const float *coef, int64_t B, const float *X,
                                        int32_t per_basis, float *Y, int64_t n_rows, int64_t F,
                                        const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_rgcn_aggr_f32";
  RgcnParams p = {};
  if (n_rows == 0) return COGDL_B200_OK;
  int rc = rgcn_setup(who, p, rowptr, colind, w, n_rows, B, F, plan);
  if (rc) return rc;
  rc = check_plan(plan, cogdl_b200_rgcn_aggr_scratch_bytes(plan->n_chunks, B, F));
  if (rc) return rc;
  CB_REQUIRE(etype && coef && X && Y, "%s: null pointer", who);
  p.etype = etype; p.coef = coef; p.X = X; p.Y = Y;
  const bool vec = (F % 4 == 0) && aligned16(X) && aligned16(Y) && (p.hub.n_chunks == 0 || aligned16(p.hub.partials));
  p.ldv = (int)(vec ? F / 4 : F);
  const cudaStream_t s = (cudaStream_t)stream;
  if (per_basis) {
    if (vec) return launch_rgcn(rgcn_fanout_kernel<float4, true>, p, s, who, "rgcn_fanout_kernel", "float4,per_basis");
    return launch_rgcn(rgcn_fanout_kernel<float, true>, p, s, who, "rgcn_fanout_kernel", "float,per_basis");
  }
  if (vec) return launch_rgcn(rgcn_fanout_kernel<float4, false>, p, s, who, "rgcn_fanout_kernel", "float4");
  return launch_rgcn(rgcn_fanout_kernel<float, false>, p, s, who, "rgcn_fanout_kernel", "float");
}

extern "C" int cogdl_b200_rgcn_edge_dot_f32(const int32_t *rowptr, const int32_t *colind, const float *w,
                                            const float *G, const float *X, float *P, int64_t n_rows, int64_t B,
                                            int64_t F, const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_rgcn_edge_dot_f32";
  RgcnParams p = {};
  if (n_rows == 0) return COGDL_B200_OK;
  int rc = rgcn_setup(who, p, rowptr, colind, w, n_rows, B, F, plan);
  if (rc) return rc;
  rc = check_plan(plan, 0);
  if (rc) return rc;
  CB_REQUIRE(G && X && P, "%s: null pointer", who);
  p.G = G; p.X = X; p.P = P;
  const bool vec = (F % 4 == 0) && aligned16(G) && aligned16(X);
  p.ldv = (int)(vec ? F / 4 : F);
  const cudaStream_t s = (cudaStream_t)stream;
  if (vec) return launch_rgcn(rgcn_edge_dot_kernel<float4>, p, s, who, "rgcn_edge_dot_kernel", "float4");
  return launch_rgcn(rgcn_edge_dot_kernel<float>, p, s, who, "rgcn_edge_dot_kernel", "float");
}

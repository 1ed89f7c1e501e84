// genconv_edge.cu -- GENConv's softmax aggregation with a linear edge encoder (DeeperGCN on ogbn-proteins;
// cogdl/layers/deepergcn_layer.py:64-93 with EdgeEncoder :168-174) for sm_90a, without any [nnz, F] tensor.
//
// The edge term of softmax_aggr.cu, A[e, f] = sum_d attr[e, d] W[f, d] (nn.Linear without bias, W [F, D]), is formed
// in registers inside the edge loop instead of being read from memory:
//   a_e[f] = fmaf(attr[e, D-1], W[f, D-1], ... fmaf(attr[e, 0], W[f, 0], 0))     (d = 0..D-1, one fixed chain)
//   m_e    = relu(X[c_e, f] + a_e[f]) + eps
// and the online softmax state, hub chunks and chunk-order merge are those of softmax_aggr.cu (softmax_aggr.cuh).
// Each lane holds the D weights of each of its channels in registers; a warp stages the D features of its 32 edges
// in its own shared memory with coalesced loads, and every lane reads them back as broadcasts.  Per edge that is
// 4 D bytes of edge data where the edge-term kernel reads 4 F.
//
// Backward, on the cached transpose (colptr, rowind, perm), as softmax_aggr_bwd_kernel: column j recomputes a_e,
// m_e, w_e and dpre_e per incoming edge (attr read through perm), accumulates dX[j] in transpose order (hub columns
// through the transpose's plan, merged in chunk order), and accumulates dW[f, d] += dpre_e[f] attr[e, d] in
// per-lane registers.  dW needs no float atomics and no per-item scratch: the grid is fixed (GE_BWD_BLOCKS, or
// fewer for a small problem), each warp strides over the work items in a static order and keeps its dW partial
// across them, the block sums its warps' partials in shared memory in warp order and writes one [F, D] partial,
// and a second small kernel sums the blocks in block order.  dW is therefore bit-identical run to run, and its
// scratch (GE_BWD_BLOCKS x F x D floats) does not grow with nnz.  Rows wider than 32 vectors run one backward
// launch per 32-vector tile (each holds only its tile's weights and dW in registers).
#include "softmax_aggr.cuh"

namespace cogdl_b200 {

constexpr int GE_MAX_D = 16;                 // widest edge feature the kernels take (registers: see DESIGN 3.18)
constexpr int GE_WARPS = 8;                  // 256-thread blocks
constexpr int GE_BWD_BLOCKS = 2 * NUM_SMS;   // fixed backward grid: the number of dW partials

struct GeFwdParams {
  SaFwdParams sa;       // sa.A unused
  const float *attr;    // [nnz, D], CSR order
  const float *Wt;      // [F, D] (nn.Linear layout)
  int D;
};

struct GeBwdParams {
  const int *colptr;
  const int *rowind;
  const int *perm;      // CSR position of transpose entry q
  const float *X;       // [n_cols, F]
  const float *attr;    // [nnz, D], CSR order
  const float *Wt;      // [F, D]
  const float *beta;
  float eps;
  const float *G;       // [n_rows, F] dL/dout
  const float *out;     // [n_rows, F]
  const float *lse2;    // [n_rows, F]
  float *dX;            // [n_cols, F] or null
  float *dW_part;       // [gridDim.x][F][D] or null
  int64_t n_cols;
  int F, FV, D;
  int tile0;            // the 32-vector tile of this launch
  HubView hub;          // plan of the transpose; partials [n_chunks][FV] vectors
};

// wr[k][d] = W[f_k, d] for the lane's channels f_k = cv * W + k; 0 past D or past the row.
template <int W, int DM>
__device__ __forceinline__ void ge_load_weights(const float *Wt, int D, int cv, bool ok, float (&wr)[W][DM]) {
#pragma unroll
  for (int k = 0; k < W; ++k)
#pragma unroll
    for (int d = 0; d < DM; ++d) wr[k][d] = ok && d < D ? __ldg(Wt + (int64_t)(cv * W + k) * D + d) : 0.f;
}

// a[k] = sum_d at[d] W[f_k, d] over d = 0..D-1, one fmaf chain from 0 (at: the edge's staged features).
template <int W, int DM>
__device__ __forceinline__ void ge_edge_term(const float *at, int D, const float (&wr)[W][DM], float (&a)[W]) {
#pragma unroll
  for (int k = 0; k < W; ++k) a[k] = 0.f;
#pragma unroll
  for (int d = 0; d < DM; ++d) {
    if (d < D) {
      const float v = at[d];
#pragma unroll
      for (int k = 0; k < W; ++k) a[k] = fmaf(v, wr[k][d], a[k]);
    }
  }
}

// One warp per work item: a hub chunk (items [0, n_chunks)) or a whole non-hub row; softmax_aggr_fwd_kernel with
// the edge term formed from the staged features.
template <int W, int DM, bool WANT_Q>
__global__ void __launch_bounds__(256, 1) genconv_edge_fwd_kernel(const GeFwdParams gp) {
  using VecT = typename SaVec<W>::T;
  constexpr int K = WANT_Q ? 4 : 3;
  constexpr int U = SA_UNROLL;
  __shared__ float s_attr[GE_WARPS][32 * DM];
  const SaFwdParams &p = gp.sa;
  const int lane = threadIdx.x & 31;
  float *sa = s_attr[threadIdx.x >> 5];
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const WorkItem w = decode_item(item, p.n_rows, p.rowptr, p.hub);
  if (!w.active) return;   // warp-uniform: past the end, or a hub row (its chunks own it)
  const float b2 = __ldg(p.beta) * SA_LOG2E;
  const VecT *X = reinterpret_cast<const VecT *>(p.X);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  const int FV = p.FV, D = gp.D;

  for (int tile0 = 0; tile0 < FV; tile0 += 32) {
    const int cv = tile0 + lane;
    const bool ok = cv < FV;
    float wr[W][DM];
    ge_load_weights<W, DM>(gp.Wt, D, cv, ok, wr);
    float M[W], S[W], T[W], Q[W];
#pragma unroll
    for (int k = 0; k < W; ++k) { M[k] = SA_M0; S[k] = 0.f; T[k] = 0.f; Q[k] = 0.f; }
    for (int e0 = w.lb; e0 < w.hb; e0 += 32) {
      const int cnt = min(32, w.hb - e0);
      const int c = lane < cnt ? ld_stream(p.colind + e0 + lane) : 0;
      const int n_at = cnt * D;
      __syncwarp();                                  // the previous batch's features are read
      for (int t = lane; t < n_at; t += 32) sa[t] = ld_stream(gp.attr + (int64_t)e0 * D + t);
      __syncwarp();
#pragma unroll 1
      for (int j = 0; j < cnt; j += U) {
        VecT xv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, c, (j + u) & 31);
          if (ok && j + u < cnt) xv[u] = ld_gather(X + (int64_t)cj * FV + cv);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (ok && j + u < cnt) {
            float xf[W], af[W];
            unpack(xv[u], xf);
            ge_edge_term<W, DM>(sa + (j + u) * D, D, wr, af);
#pragma unroll
            for (int k = 0; k < W; ++k) sa_step<WANT_Q>(relu_nan(xf[k] + af[k]) + p.eps, b2, M[k], S[k], T[k], Q[k]);
          }
        }
      }
    }
    if (ok && w.is_chunk) {
      VecT *pp = P + (int64_t)w.slot * K * FV + cv;
      st_cg(pp, pack(M));
      st_cg(pp + FV, pack(S));
      st_cg(pp + 2 * FV, pack(T));
      if (WANT_Q) st_cg(pp + 3 * FV, pack(Q));
    } else if (ok) {
      sa_finish<W, WANT_Q>(p, (int64_t)w.row * FV + cv, M, S, T, Q, w.hb > w.lb);
    }
  }
  if (w.is_chunk && hub_arrive_last<32>(w, p.hub, lane)) {
    for (int cv = lane; cv < FV; cv += 32) {
      float M[W], S[W], T[W], Q[W];
#pragma unroll
      for (int k = 0; k < W; ++k) { M[k] = SA_M0; S[k] = 0.f; T[k] = 0.f; Q[k] = 0.f; }
      for (int q = 0; q < w.n_row_chunks; ++q) {   // chunk order: deterministic
        const VecT *pp = P + (int64_t)(w.first + q) * K * FV + cv;
        float Mc[W], Sc[W], Tc[W], Qc[W];
        unpack(ld_cg(pp), Mc);
        unpack(ld_cg(pp + FV), Sc);
        unpack(ld_cg(pp + 2 * FV), Tc);
        if (WANT_Q) unpack(ld_cg(pp + 3 * FV), Qc);
#pragma unroll
        for (int k = 0; k < W; ++k) sa_merge(Mc[k], Sc[k], Tc[k], WANT_Q ? Qc[k] : 0.f, M[k], S[k], T[k], Q[k]);
      }
      sa_finish<W, WANT_Q>(p, (int64_t)w.row * FV + cv, M, S, T, Q, true);
    }
  }
}

// One 32-vector tile of the backward.  Warps stride over the transpose's work items in a static order; dX as in
// softmax_aggr_bwd_kernel, dW summed per lane across the warp's items, then over the block's warps in warp order.
template <int W, int DM>
__global__ void __launch_bounds__(256, 1) genconv_edge_bwd_kernel(const GeBwdParams p) {
  using VecT = typename SaVec<W>::T;
  constexpr int U = SA_UNROLL;
  constexpr int WD = W * DM;
  __shared__ float s_attr[GE_WARPS][32 * DM];
  __shared__ float s_dw[32][WD + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *sa = s_attr[warp];
  const float beta = __ldg(p.beta);
  const float b2 = beta * SA_LOG2E;
  const VecT *X = reinterpret_cast<const VecT *>(p.X);
  const VecT *G = reinterpret_cast<const VecT *>(p.G);
  const VecT *O = reinterpret_cast<const VecT *>(p.out);
  const VecT *L = reinterpret_cast<const VecT *>(p.lse2);
  VecT *dX = reinterpret_cast<VecT *>(p.dX);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  const int FV = p.FV, D = p.D;
  const bool want_dw = p.dW_part != nullptr;
  const int cv = p.tile0 + lane;
  const bool ok = cv < FV;
  float wr[W][DM], dw[W][DM];
  ge_load_weights<W, DM>(p.Wt, D, cv, ok, wr);
#pragma unroll
  for (int k = 0; k < W; ++k)
#pragma unroll
    for (int d = 0; d < DM; ++d) dw[k][d] = 0.f;

  const int64_t n_items = (int64_t)p.hub.n_chunks + p.n_cols;
  const int64_t stride = (int64_t)gridDim.x * GE_WARPS;
  for (int64_t item = (int64_t)blockIdx.x * GE_WARPS + warp; item < n_items; item += stride) {
    const WorkItem w = decode_item(item, p.n_cols, p.colptr, p.hub);
    if (!w.active) continue;   // warp-uniform: a hub column (its chunks own it)
    float xj[W], acc[W];
#pragma unroll
    for (int k = 0; k < W; ++k) { xj[k] = 0.f; acc[k] = 0.f; }
    if (ok) unpack(ld_gather(X + (int64_t)w.row * FV + cv), xj);
    for (int e0 = w.lb; e0 < w.hb; e0 += 32) {
      const int cnt = min(32, w.hb - e0);
      int r = 0, pe = 0;
      if (lane < cnt) {
        r = ld_stream(p.rowind + e0 + lane);
        pe = ld_stream(p.perm + e0 + lane);
      }
      // stage the features of the batch's edges: entry t is attr[perm[e0 + t / D], t % D]
      const int n_at = cnt * D;
      __syncwarp();
      for (int t0 = 0; t0 < n_at; t0 += 32) {
        const int t = t0 + lane;
        const int e = t / D;
        const int pv = __shfl_sync(FULL, pe, e & 31);
        if (t < n_at) sa[t] = ld_stream(p.attr + (int64_t)pv * D + (t - e * D));
      }
      __syncwarp();
#pragma unroll 1
      for (int j = 0; j < cnt; j += U) {
        VecT lv[U], gv[U], ov[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int rj = __shfl_sync(FULL, r, (j + u) & 31);
          if (ok && j + u < cnt) {
            const int64_t ro = (int64_t)rj * FV + cv;
            lv[u] = ld_gather(L + ro);
            gv[u] = ld_gather(G + ro);
            ov[u] = ld_gather(O + ro);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (ok && j + u < cnt) {
            const float *at = sa + (j + u) * D;
            float lf[W], gf[W], of[W], af[W], da[W];
            unpack(lv[u], lf);
            unpack(gv[u], gf);
            unpack(ov[u], of);
            ge_edge_term<W, DM>(at, D, wr, af);
#pragma unroll
            for (int k = 0; k < W; ++k) {
              const float pre = xj[k] + af[k];
              const float m = relu_nan(pre) + p.eps;
              const float wgt = exp2f(fmaf(m, b2, -lf[k]));
              const float dm = wgt * gf[k] * fmaf(beta, m - of[k], 1.f);
              da[k] = pre <= 0.f ? 0.f : dm;          // torch's relu backward: a NaN pre passes its gradient
              acc[k] += da[k];
            }
            if (want_dw) {
#pragma unroll
              for (int d = 0; d < DM; ++d) {
                if (d < D) {
                  const float v = at[d];
#pragma unroll
                  for (int k = 0; k < W; ++k) dw[k][d] = fmaf(da[k], v, dw[k][d]);
                }
              }
            }
          }
        }
      }
    }
    if (dX) {
      if (ok && w.is_chunk) st_cg(P + (int64_t)w.slot * FV + cv, pack(acc));
      else if (ok) st_stream(dX + (int64_t)w.row * FV + cv, pack(acc));
      if (w.is_chunk && hub_arrive_last<32>(w, p.hub, lane) && ok) {
        const VecT *pp = P + (int64_t)w.first * FV + cv;
        float s[W], t[W];
        unpack(ld_cg(pp), s);
        for (int q = 1; q < w.n_row_chunks; ++q) {   // chunk order: deterministic
          unpack(ld_cg(pp + (int64_t)q * FV), t);
#pragma unroll
          for (int k = 0; k < W; ++k) s[k] += t[k];
        }
        st_stream(dX + (int64_t)w.row * FV + cv, pack(s));
      }
    }
  }
  if (!want_dw) return;   // block-uniform
  // the block's dW tile: warps 0..7 in order into shared memory, then one [32 W, D] slice of this block's partial
#pragma unroll 1
  for (int wi = 0; wi < GE_WARPS; ++wi) {
    if (warp == wi) {
#pragma unroll
      for (int k = 0; k < W; ++k)
#pragma unroll
        for (int d = 0; d < DM; ++d) s_dw[lane][k * DM + d] = wi == 0 ? dw[k][d] : s_dw[lane][k * DM + d] + dw[k][d];
    }
    __syncthreads();
  }
  const int n_f = min(32, FV - p.tile0) * W;          // channels of this tile
  float *part = p.dW_part + ((int64_t)blockIdx.x * p.F + (int64_t)p.tile0 * W) * D;
  for (int t = threadIdx.x; t < n_f * D; t += blockDim.x) {
    const int f = t / D, d = t - f * D;
    part[t] = s_dw[f / W][(f % W) * DM + d];
  }
}

// dW[i] = sum over the n_blocks partials in block order, i over the F * D entries.
__global__ void __launch_bounds__(256) genconv_edge_dw_reduce_kernel(const float *part, int n_blocks, int64_t FD,
                                                                     float *dW) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= FD) return;
  float s = part[i];
  for (int b = 1; b < n_blocks; ++b) s += part[(int64_t)b * FD + i];
  dW[i] = s;
}

template <int W, int DM>
static void launch_fwd(const GeFwdParams &p, bool want_q, unsigned blocks, cudaStream_t s) {
  if (want_q) genconv_edge_fwd_kernel<W, DM, true><<<blocks, 256, 0, s>>>(p);
  else genconv_edge_fwd_kernel<W, DM, false><<<blocks, 256, 0, s>>>(p);
}

template <int W>
static void launch_fwd_d(const GeFwdParams &p, bool want_q, unsigned blocks, cudaStream_t s) {
  if (p.D <= 8) launch_fwd<W, 8>(p, want_q, blocks, s);
  else launch_fwd<W, 16>(p, want_q, blocks, s);
}

template <int W>
static void launch_bwd_d(const GeBwdParams &p, unsigned blocks, cudaStream_t s) {
  if (p.D <= 8) genconv_edge_bwd_kernel<W, 8><<<blocks, 256, 0, s>>>(p);
  else genconv_edge_bwd_kernel<W, 16><<<blocks, 256, 0, s>>>(p);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_genconv_edge_dw_scratch_bytes(int64_t F, int64_t D) {
  return F > 0 && D > 0 ? (int64_t)GE_BWD_BLOCKS * F * D * 4 : 0;
}

// only dX's hub columns use the partials
extern "C" int64_t cogdl_b200_genconv_edge_bwd_scratch_bytes(int64_t n_chunks, int64_t F, int32_t want_dx) {
  return want_dx ? cogdl_b200_softmax_aggr_bwd_scratch_bytes(n_chunks, F) : 0;
}

extern "C" int cogdl_b200_genconv_edge_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *X,
                                               const float *attr, const float *W, int64_t D, const float *beta,
                                               float eps, float *out, float *lse2, float *Q, int64_t n_rows, int64_t F,
                                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && F >= 0, "cogdl_b200_genconv_edge_fwd_f32: negative size");
  CB_REQUIRE(D >= 1 && D <= GE_MAX_D, "cogdl_b200_genconv_edge_fwd_f32: D = %lld, must be in [1, %d]", (long long)D,
             GE_MAX_D);
  if (n_rows == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && X && attr && W && beta && out, "cogdl_b200_genconv_edge_fwd_f32: null pointer");
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "cogdl_b200_genconv_edge_fwd_f32: sizes must fit int32");
  const int64_t n_chunks = plan && plan->chunk_edges > 0 ? plan->n_chunks : 0;
  int rc = check_plan(plan, cogdl_b200_softmax_aggr_scratch_bytes(n_chunks, F));
  if (rc) return rc;
  GeFwdParams p;
  SaFwdParams &s = p.sa;
  s.rowptr = rowptr; s.colind = colind; s.X = X; s.A = nullptr; s.beta = beta; s.eps = eps;
  s.out = out; s.lse2 = lse2; s.Q = Q; s.n_rows = n_rows;
  s.hub = hub_view(plan);
  p.attr = attr; p.Wt = W; p.D = (int)D;
  const bool vec = F % 4 == 0 && aligned16(X) && aligned16(out) && (!lse2 || aligned16(lse2)) && (!Q || aligned16(Q)) &&
                   (n_chunks == 0 || aligned16(s.hub.partials));
  s.FV = (int)(vec ? F / 4 : F);
  const int64_t blocks = ceil_div((n_chunks + n_rows) * 32, 256);
  CB_REQUIRE(blocks <= 0x7fffffffLL, "cogdl_b200_genconv_edge_fwd_f32: problem too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;
  if (vec) launch_fwd_d<4>(p, Q != nullptr, (unsigned)blocks, st);
  else launch_fwd_d<1>(p, Q != nullptr, (unsigned)blocks, st);
  note_kernel("cogdl_b200::genconv_edge_fwd_kernel<%s,DM=%d,%s>", vec ? "float4" : "float", D <= 8 ? 8 : 16,
              Q ? "Q" : "no_Q");
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_genconv_edge_bwd_f32(const int32_t *colptr, const int32_t *rowind, const int32_t *perm,
                                               const float *X, const float *attr, const float *W, int64_t D,
                                               const float *beta, float eps, const float *G, const float *out,
                                               const float *lse2, float *dX, float *dW, float *dw_scratch,
                                               int64_t dw_scratch_bytes, int64_t n_cols, int64_t F,
                                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_cols >= 0 && F >= 0, "cogdl_b200_genconv_edge_bwd_f32: negative size");
  CB_REQUIRE(D >= 1 && D <= GE_MAX_D, "cogdl_b200_genconv_edge_bwd_f32: D = %lld, must be in [1, %d]", (long long)D,
             GE_MAX_D);
  CB_REQUIRE(dX || dW, "cogdl_b200_genconv_edge_bwd_f32: neither dX nor dW asked for");
  CB_REQUIRE(!dW || (dw_scratch && dw_scratch_bytes >= cogdl_b200_genconv_edge_dw_scratch_bytes(F, D)),
             "cogdl_b200_genconv_edge_bwd_f32: dW needs %lld bytes of dw_scratch, got %lld",
             (long long)cogdl_b200_genconv_edge_dw_scratch_bytes(F, D), (long long)(dw_scratch ? dw_scratch_bytes : 0));
  if (F == 0) return COGDL_B200_OK;
  if (n_cols == 0) {   // no columns, no edges: dW = 0
    if (dW) CB_CUDA(cudaMemsetAsync(dW, 0, (size_t)(F * D) * sizeof(float), (cudaStream_t)stream));
    return COGDL_B200_OK;
  }
  CB_REQUIRE(colptr && rowind && perm && X && attr && W && beta && G && out && lse2,
             "cogdl_b200_genconv_edge_bwd_f32: null pointer");
  CB_REQUIRE(n_cols < 0x7fffffffLL && F < 0x7fffffffLL, "cogdl_b200_genconv_edge_bwd_f32: sizes must fit int32");
  const int64_t n_chunks = plan && plan->chunk_edges > 0 ? plan->n_chunks : 0;
  int rc = check_plan(plan, cogdl_b200_genconv_edge_bwd_scratch_bytes(n_chunks, F, dX != nullptr));
  if (rc) return rc;
  GeBwdParams p;
  p.colptr = colptr; p.rowind = rowind; p.perm = perm; p.X = X; p.attr = attr; p.Wt = W; p.beta = beta; p.eps = eps;
  p.G = G; p.out = out; p.lse2 = lse2; p.dX = dX; p.dW_part = dW ? dw_scratch : nullptr; p.n_cols = n_cols;
  p.F = (int)F; p.D = (int)D;
  p.hub = hub_view(plan);
  const bool vec = F % 4 == 0 && aligned16(X) && aligned16(G) && aligned16(out) && aligned16(lse2) &&
                   (!dX || aligned16(dX)) && (n_chunks == 0 || !dX || aligned16(p.hub.partials));
  p.FV = (int)(vec ? F / 4 : F);
  const int64_t items = ceil_div(n_chunks + n_cols, GE_WARPS);
  const int64_t blocks = items < GE_BWD_BLOCKS ? items : GE_BWD_BLOCKS;
  cudaStream_t st = (cudaStream_t)stream;
  for (int tile0 = 0; tile0 < p.FV; tile0 += 32) {   // stream order: a tile's hub merges reset the counters
    p.tile0 = tile0;
    if (vec) launch_bwd_d<4>(p, (unsigned)blocks, st);
    else launch_bwd_d<1>(p, (unsigned)blocks, st);
    CB_LAUNCH_CHECK();
  }
  note_kernel("cogdl_b200::genconv_edge_bwd_kernel<%s,DM=%d>", vec ? "float4" : "float", D <= 8 ? 8 : 16);
  if (dW) {
    genconv_edge_dw_reduce_kernel<<<(unsigned)ceil_div(F * D, 256), 256, 0, st>>>(dw_scratch, (int)blocks, F * D, dW);
    append_kernel_note(" + cogdl_b200::genconv_edge_dw_reduce_kernel");
    CB_LAUNCH_CHECK();
  }
  return COGDL_B200_OK;
}

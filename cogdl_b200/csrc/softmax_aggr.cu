// softmax_aggr.cu -- GENConv's softmax aggregation (DeeperGCN, cogdl/layers/deepergcn_layer.py:64-93) for sm_90a.
//
// Per output row i, channel f, over the CSR edges e = (i, c_e):
//   m_e   = relu(X[c_e,f] + A[e,f]) + eps              (A: optional edge term, [nnz, F] in CSR order)
//   out_i = sum_e w_e m_e,   w_e = 2^(b2 m_e - lse2_i),   b2 = beta * log2(e),   lse2_i = log2 sum_e 2^(b2 m_e)
// i.e. softmax_e(beta * m_e) weighted by m_e, with the logits kept in base 2 so every exponential is one ex2.
// The reference forms m, beta*m, the softmax and the product as four [nnz, F] tensors and scatter_adds them
// with float atomics; here each lane owns channels of the row and keeps an online (M, S, T[, Q]) in registers:
//   M = max b2 m,  S = sum 2^(b2 m - M),  T = sum 2^(b2 m - M) m,  Q = sum 2^(b2 m - M) m^2
// with ONE exponential per edge and channel (2^-|d| rescales either the sum or the new term).  Nothing
// edge-sized is written.  Hub rows are cut into the plan's chunks, each writing its partial (M, S, T[, Q]);
// the last chunk to arrive merges them in chunk order, so results are bit-reproducible run to run.
//
// Backward, on the cached transpose (colptr, rowind, perm): column j holds X[j] in registers and walks its
// incoming edges (i, e).  Per edge it recomputes m_e and w_e from the saved lse2_i and
//   dm_e = g_i w_e (1 + beta (m_e - out_i)),   dpre_e = dm_e [X[j] + A_e > 0]
// accumulates dX[j] = sum dpre_e in transpose order (hub columns through the transpose's plan, merged in chunk
// order) and, with an edge term, writes dA[perm[q]] = dpre_e (each slot once).  d beta = sum g (Q - out^2) is a
// dense reduction over the saved Q, done by the caller.
#include "softmax_aggr.cuh"   // the online (M, S, T[, Q]) state, shared with genconv_edge.cu

namespace cogdl_b200 {

// One warp per work item: a hub chunk (items [0, n_chunks)) or a whole non-hub row.
template <int W, bool HAS_A, bool WANT_Q>
__global__ void __launch_bounds__(256) softmax_aggr_fwd_kernel(const SaFwdParams p) {
  using VecT = typename SaVec<W>::T;
  constexpr int K = WANT_Q ? 4 : 3;
  constexpr int U = SA_UNROLL;
  const int lane = threadIdx.x & 31;
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const WorkItem w = decode_item(item, p.n_rows, p.rowptr, p.hub);
  if (!w.active) return;   // warp-uniform: past the end, or a hub row (its chunks own it)
  const float b2 = __ldg(p.beta) * SA_LOG2E;
  const VecT *X = reinterpret_cast<const VecT *>(p.X);
  const VecT *A = reinterpret_cast<const VecT *>(p.A);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  const int FV = p.FV;

  for (int tile0 = 0; tile0 < FV; tile0 += 32) {
    const int cv = tile0 + lane;
    const bool ok = cv < FV;
    float M[W], S[W], T[W], Q[W];
#pragma unroll
    for (int k = 0; k < W; ++k) { M[k] = SA_M0; S[k] = 0.f; T[k] = 0.f; Q[k] = 0.f; }
    for (int e0 = w.lb; e0 < w.hb; e0 += 32) {
      const int cnt = min(32, w.hb - e0);
      const int c = lane < cnt ? ld_stream(p.colind + e0 + lane) : 0;
#pragma unroll 1
      for (int j = 0; j < cnt; j += U) {
        VecT xv[U], av[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, c, (j + u) & 31);
          if (ok && j + u < cnt) {
            xv[u] = ld_gather(X + (int64_t)cj * FV + cv);
            if (HAS_A) av[u] = ld_edge(A + (int64_t)(e0 + j + u) * FV + cv);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (ok && j + u < cnt) {
            float xf[W], af[W];
            unpack(xv[u], xf);
            if (HAS_A) unpack(av[u], af);
#pragma unroll
            for (int k = 0; k < W; ++k) {
              const float pre = HAS_A ? xf[k] + af[k] : xf[k];
              sa_step<WANT_Q>(relu_nan(pre) + p.eps, b2, M[k], S[k], T[k], Q[k]);
            }
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

struct SaBwdParams {
  const int *colptr;
  const int *rowind;
  const int *perm;      // CSR position of transpose entry q (needed with an edge term)
  const float *X;       // [n_cols, F]
  const float *A;       // [nnz, F] or null
  const float *beta;
  float eps;
  const float *G;       // [n_rows, F] dL/dout
  const float *out;     // [n_rows, F]
  const float *lse2;    // [n_rows, F]
  float *dX;            // [n_cols, F]
  float *dA;            // [nnz, F] or null
  int64_t n_cols;
  int FV;
  HubView hub;          // plan of the transpose; partials [n_chunks][FV] vectors
};

template <int W, bool HAS_A>
__global__ void __launch_bounds__(256) softmax_aggr_bwd_kernel(const SaBwdParams p) {
  using VecT = typename SaVec<W>::T;
  constexpr int U = SA_UNROLL;
  const int lane = threadIdx.x & 31;
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const WorkItem w = decode_item(item, p.n_cols, p.colptr, p.hub);
  if (!w.active) return;
  const float beta = __ldg(p.beta);
  const float b2 = beta * SA_LOG2E;
  const VecT *X = reinterpret_cast<const VecT *>(p.X);
  const VecT *A = reinterpret_cast<const VecT *>(p.A);
  const VecT *G = reinterpret_cast<const VecT *>(p.G);
  const VecT *O = reinterpret_cast<const VecT *>(p.out);
  const VecT *L = reinterpret_cast<const VecT *>(p.lse2);
  VecT *dA = reinterpret_cast<VecT *>(p.dA);
  VecT *dX = reinterpret_cast<VecT *>(p.dX);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  const int FV = p.FV;

  for (int tile0 = 0; tile0 < FV; tile0 += 32) {
    const int cv = tile0 + lane;
    const bool ok = cv < FV;
    float xj[W], acc[W];
#pragma unroll
    for (int k = 0; k < W; ++k) { xj[k] = 0.f; acc[k] = 0.f; }
    if (ok) unpack(ld_gather(X + (int64_t)w.row * FV + cv), xj);
    for (int e0 = w.lb; e0 < w.hb; e0 += 32) {
      const int cnt = min(32, w.hb - e0);
      int r = 0, pe = 0;
      if (lane < cnt) {
        r = ld_stream(p.rowind + e0 + lane);
        if (HAS_A) pe = ld_stream(p.perm + e0 + lane);
      }
#pragma unroll 1
      for (int j = 0; j < cnt; j += U) {
        VecT lv[U], gv[U], ov[U], av[U];
        int pj[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int rj = __shfl_sync(FULL, r, (j + u) & 31);
          pj[u] = HAS_A ? __shfl_sync(FULL, pe, (j + u) & 31) : 0;
          if (ok && j + u < cnt) {
            const int64_t ro = (int64_t)rj * FV + cv;
            lv[u] = ld_gather(L + ro);
            gv[u] = ld_gather(G + ro);
            ov[u] = ld_gather(O + ro);
            if (HAS_A) av[u] = ld_edge(A + (int64_t)pj[u] * FV + cv);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (ok && j + u < cnt) {
            float lf[W], gf[W], of[W], af[W], da[W];
            unpack(lv[u], lf);
            unpack(gv[u], gf);
            unpack(ov[u], of);
            if (HAS_A) unpack(av[u], af);
#pragma unroll
            for (int k = 0; k < W; ++k) {
              const float pre = HAS_A ? xj[k] + af[k] : xj[k];
              const float m = relu_nan(pre) + p.eps;
              const float wgt = exp2f(fmaf(m, b2, -lf[k]));
              const float dm = wgt * gf[k] * fmaf(beta, m - of[k], 1.f);
              da[k] = pre <= 0.f ? 0.f : dm;          // torch's relu backward: a NaN pre passes its gradient
              acc[k] += da[k];
            }
            if (HAS_A && dA) __stcs(dA + (int64_t)pj[u] * FV + cv, pack(da));
          }
        }
      }
    }
    if (ok && w.is_chunk) st_cg(P + (int64_t)w.slot * FV + cv, pack(acc));
    else if (ok) st_stream(dX + (int64_t)w.row * FV + cv, pack(acc));
  }
  if (w.is_chunk && hub_arrive_last<32>(w, p.hub, lane)) {
    for (int cv = lane; cv < FV; cv += 32) {
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

static int64_t sa_blocks(int64_t n_chunks, int64_t n_rows) { return ceil_div((n_chunks + n_rows) * 32, 256); }

template <int W, bool HAS_A>
static void launch_fwd(const SaFwdParams &p, bool want_q, unsigned blocks, cudaStream_t s) {
  if (want_q) softmax_aggr_fwd_kernel<W, HAS_A, true><<<blocks, 256, 0, s>>>(p);
  else softmax_aggr_fwd_kernel<W, HAS_A, false><<<blocks, 256, 0, s>>>(p);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_softmax_aggr_scratch_bytes(int64_t n_chunks, int64_t F) {
  return n_chunks > 0 && F > 0 ? n_chunks * F * 16 : 0;
}

extern "C" int64_t cogdl_b200_softmax_aggr_bwd_scratch_bytes(int64_t n_chunks, int64_t F) {
  return n_chunks > 0 && F > 0 ? n_chunks * F * 4 : 0;
}

extern "C" int cogdl_b200_softmax_aggr_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *X,
                                               const float *edge_term, const float *beta, float eps, float *out,
                                               float *lse2, float *Q, int64_t n_rows, int64_t F,
                                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_rows >= 0 && F >= 0, "cogdl_b200_softmax_aggr_fwd_f32: negative size");
  if (n_rows == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && X && beta && out, "cogdl_b200_softmax_aggr_fwd_f32: null pointer");
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "cogdl_b200_softmax_aggr_fwd_f32: sizes must fit int32");
  const int64_t n_chunks = plan && plan->chunk_edges > 0 ? plan->n_chunks : 0;
  int rc = check_plan(plan, cogdl_b200_softmax_aggr_scratch_bytes(n_chunks, F));
  if (rc) return rc;
  SaFwdParams p;
  p.rowptr = rowptr; p.colind = colind; p.X = X; p.A = edge_term; p.beta = beta; p.eps = eps;
  p.out = out; p.lse2 = lse2; p.Q = Q; p.n_rows = n_rows;
  p.hub = hub_view(plan);
  const bool vec = F % 4 == 0 && aligned16(X) && aligned16(out) && (!edge_term || aligned16(edge_term)) &&
                   (!lse2 || aligned16(lse2)) && (!Q || aligned16(Q)) && (n_chunks == 0 || aligned16(p.hub.partials));
  p.FV = (int)(vec ? F / 4 : F);
  const int64_t blocks = sa_blocks(n_chunks, n_rows);
  CB_REQUIRE(blocks <= 0x7fffffffLL, "cogdl_b200_softmax_aggr_fwd_f32: problem too large for one launch");
  cudaStream_t s = (cudaStream_t)stream;
  if (vec) {
    if (edge_term) launch_fwd<4, true>(p, Q != nullptr, (unsigned)blocks, s);
    else launch_fwd<4, false>(p, Q != nullptr, (unsigned)blocks, s);
  } else {
    if (edge_term) launch_fwd<1, true>(p, Q != nullptr, (unsigned)blocks, s);
    else launch_fwd<1, false>(p, Q != nullptr, (unsigned)blocks, s);
  }
  note_kernel("cogdl_b200::softmax_aggr_fwd_kernel<%s,%s,%s>", vec ? "float4" : "float",
              edge_term ? "edge_term" : "no_edge_term", Q ? "Q" : "no_Q");
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_softmax_aggr_bwd_f32(const int32_t *colptr, const int32_t *rowind, const int32_t *perm,
                                               const float *X, const float *edge_term, const float *beta, float eps,
                                               const float *G, const float *out, const float *lse2, float *dX,
                                               float *d_edge_term, int64_t n_cols, int64_t F,
                                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  CB_REQUIRE(n_cols >= 0 && F >= 0, "cogdl_b200_softmax_aggr_bwd_f32: negative size");
  if (n_cols == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(colptr && rowind && X && beta && G && out && lse2 && dX, "cogdl_b200_softmax_aggr_bwd_f32: null pointer");
  CB_REQUIRE(!edge_term || perm, "cogdl_b200_softmax_aggr_bwd_f32: an edge term needs the transpose's perm");
  CB_REQUIRE(!d_edge_term || edge_term, "cogdl_b200_softmax_aggr_bwd_f32: d_edge_term without an edge term");
  CB_REQUIRE(n_cols < 0x7fffffffLL && F < 0x7fffffffLL, "cogdl_b200_softmax_aggr_bwd_f32: sizes must fit int32");
  const int64_t n_chunks = plan && plan->chunk_edges > 0 ? plan->n_chunks : 0;
  int rc = check_plan(plan, cogdl_b200_softmax_aggr_bwd_scratch_bytes(n_chunks, F));
  if (rc) return rc;
  SaBwdParams p;
  p.colptr = colptr; p.rowind = rowind; p.perm = perm; p.X = X; p.A = edge_term; p.beta = beta; p.eps = eps;
  p.G = G; p.out = out; p.lse2 = lse2; p.dX = dX; p.dA = d_edge_term; p.n_cols = n_cols;
  p.hub = hub_view(plan);
  const bool vec = F % 4 == 0 && aligned16(X) && aligned16(G) && aligned16(out) && aligned16(lse2) && aligned16(dX) &&
                   (!edge_term || aligned16(edge_term)) && (!d_edge_term || aligned16(d_edge_term)) &&
                   (n_chunks == 0 || aligned16(p.hub.partials));
  p.FV = (int)(vec ? F / 4 : F);
  const int64_t blocks = sa_blocks(n_chunks, n_cols);
  CB_REQUIRE(blocks <= 0x7fffffffLL, "cogdl_b200_softmax_aggr_bwd_f32: problem too large for one launch");
  cudaStream_t s = (cudaStream_t)stream;
  if (vec) {
    if (edge_term) softmax_aggr_bwd_kernel<4, true><<<(unsigned)blocks, 256, 0, s>>>(p);
    else softmax_aggr_bwd_kernel<4, false><<<(unsigned)blocks, 256, 0, s>>>(p);
  } else {
    if (edge_term) softmax_aggr_bwd_kernel<1, true><<<(unsigned)blocks, 256, 0, s>>>(p);
    else softmax_aggr_bwd_kernel<1, false><<<(unsigned)blocks, 256, 0, s>>>(p);
  }
  note_kernel("cogdl_b200::softmax_aggr_bwd_kernel<%s,%s>", vec ? "float4" : "float", edge_term ? "edge_term" : "no_edge_term");
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

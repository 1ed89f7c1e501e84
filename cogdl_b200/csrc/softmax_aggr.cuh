// softmax_aggr.cuh -- the online softmax state of GENConv's aggregation, shared by softmax_aggr.cu (edge term read
// from an [nnz, F] tensor) and genconv_edge.cu (edge term computed from the edge features in registers).
//
// Per channel a lane keeps (M, S, T[, Q]) over the edges it has seen, in base 2:
//   M = max b2 m,  S = sum 2^(b2 m - M),  T = sum 2^(b2 m - M) m,  Q = sum 2^(b2 m - M) m^2
// with ONE exponential per edge and channel (2^-|d| rescales either the sum or the new term).
#pragma once
#include "common.cuh"

#include <math_constants.h>

#include <cfloat>

namespace cogdl_b200 {

constexpr float SA_LOG2E = 1.4426950408889634f;
// The running max M starts at -FLT_MAX, not -inf: a -inf logit (a negative beta times a message past ~2^127) then
// gives d = -inf and weight 0 wherever it falls, where -inf - (-inf) would make the row NaN.
constexpr float SA_M0 = -FLT_MAX;
constexpr int SA_UNROLL = 4;   // gathers in flight per lane (8 measured slower: 573-625 vs 472-515 us, arxiv F = 128)

template <int W> struct SaVec;
template <> struct SaVec<1> { using T = float; };
template <> struct SaVec<4> { using T = float4; };

__device__ __forceinline__ void unpack(const float &v, float (&o)[1]) { o[0] = v; }
__device__ __forceinline__ void unpack(const float4 &v, float (&o)[4]) { o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; }
__device__ __forceinline__ float pack(const float (&o)[1]) { return o[0]; }
__device__ __forceinline__ float4 pack(const float (&o)[4]) { return make_float4(o[0], o[1], o[2], o[3]); }
__device__ __forceinline__ float ld_edge(const float *p) { return __ldcs(p); }
__device__ __forceinline__ float4 ld_edge(const float4 *p) { return __ldcs(p); }

struct SaFwdParams {
  const int *rowptr;
  const int *colind;
  const float *X;      // [n_cols, F]
  const float *A;      // [nnz, F] or null
  const float *beta;   // device scalar
  float eps;
  float *out;          // [n_rows, F]
  float *lse2;         // [n_rows, F] or null
  float *Q;            // [n_rows, F], written iff the kernel is instantiated with WANT_Q
  int64_t n_rows;
  int FV;              // row length in vectors
  HubView hub;         // partials: [n_chunks][3 or 4][FV] vectors
};

// One edge into the online state.  M = SA_M0 on entry gives d > 0 and S = 1, T = m, M = z for any z above -FLT_MAX;
// z = -inf gives e = 0 and adds nothing (T += 0 * m: NaN for an infinite m, as exp(-inf) * m is in the softmax).
template <bool WANT_Q>
__device__ __forceinline__ void sa_step(float m, float b2, float &M, float &S, float &T, float &Q) {
  const float z = m * b2;
  const float d = z - M;
  const float e = exp2f(-fabsf(d));
  if (d > 0.f) {
    S = fmaf(S, e, 1.f);
    T = fmaf(T, e, m);
    if (WANT_Q) Q = fmaf(Q, e, m * m);
    M = z;
  } else {
    S += e;
    T = fmaf(e, m, T);
    if (WANT_Q) Q = fmaf(e * m, m, Q);
  }
}

// Fold a chunk's partial state into (M, S, T, Q); M = SA_M0 on entry takes the partial as it is (a chunk's M is at
// least SA_M0, so no -inf - (-inf) forms here either).
__device__ __forceinline__ void sa_merge(float Mc, float Sc, float Tc, float Qc, float &M, float &S, float &T, float &Q) {
  const float Mn = fmaxf(M, Mc);
  const float a = exp2f(M - Mn), b = exp2f(Mc - Mn);
  S = fmaf(S, a, Sc * b);
  T = fmaf(T, a, Tc * b);
  Q = fmaf(Q, a, Qc * b);
  M = Mn;
}

template <int W, bool WANT_Q>
__device__ __forceinline__ void sa_finish(const SaFwdParams &p, int64_t off, const float (&M)[W], const float (&S)[W],
                                          const float (&T)[W], const float (&Q)[W], bool any) {
  using VecT = typename SaVec<W>::T;
  float o[W], l[W], q[W];
#pragma unroll
  for (int k = 0; k < W; ++k) {
    // `any` comes from the CSR: degree-0 rows give out = 0 (a scatter_add of nothing), while a row whose logits are
    // all -inf has S = 0 and gives T / S = NaN, as the softmax does.  A +Inf logit is its row's max, and
    // exp(z - max) = exp(Inf - Inf) is NaN in the softmax this restates: the online state counted it as 1, so the
    // row's sums are replaced by NaN here
    const float s = M[k] < CUDART_INF_F ? S[k] : CUDART_NAN_F;
    o[k] = any ? T[k] / s : 0.f;
    l[k] = any ? M[k] + log2f(s) : 0.f;
    q[k] = any ? Q[k] / s : 0.f;
  }
  st_stream(reinterpret_cast<VecT *>(p.out) + off, pack(o));
  if (p.lse2) st_stream(reinterpret_cast<VecT *>(p.lse2) + off, pack(l));
  if (WANT_Q) st_stream(reinterpret_cast<VecT *>(p.Q) + off, pack(q));
}

}  // namespace cogdl_b200

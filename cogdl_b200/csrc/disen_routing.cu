// disen_routing.cu -- one neighbourhood-routing step of DisenGCN (cogdl/layers/disengcn_layer.py:40-91) for sm_90a.
//
// A row of F = K*d floats is K channels of d; channel k is columns [k*d, (k+1)*d).  Given the normalised features
// c (unit norm per node and channel) and the current routing state q, per row i, channel k, over the CSR edges
// e = (i, j):
//   s_e = (q_i,k . c_j,k) / tau,   w_e = softmax over row i's edges of s_e,   a_i,k = sum_e w_e c_j,k
//   u_i,k = a_i,k + c_i,k,         out_i,k = u_i,k / |u_i,k|                 (degree-0 rows: u = c)
// The reference forms h_dst[row], h_src[col], their product, the index_select and the weighted messages as five
// [E, K, d] tensors plus an int64 [K, E, d] index per iteration and scatter_adds with float atomics.  Here the
// L = d / W lanes of a channel (W = 4 floats per lane with float4 vectors, else 1) form an aligned group; the dot
// product is a __shfl_xor butterfly inside it, and every lane keeps an online softmax (M, S) of its channel in base
// 2 (one ex2 per edge and channel) beside its part of sum 2^(z - M) c_j.  Rows narrower than a warp share it
// (GROUP lanes per row, as spmm_kernel does); rows wider than 32 vectors loop over 32-vector tiles.  Hub rows are
// cut into the plan's chunks, each writes its partial (acc, M, S), and the last chunk to arrive merges them in chunk
// order: no float atomics, bit-reproducible run to run.  Nothing edge-sized is written.
//
// Backward, given g = dL/dout and the forward's lse2 = log2 sum_e 2^(s_e log2 e) and r = |u| ([n, K]):
//   g_u = (g - out (out . g)) / r,   t_e = g_u,i . c_j,   D_i = sum_e w_e t_e  (= g_u,i . a_i)
//   dq_i = sum_e w_e (t_e - D_i) c_j / tau = (sum_e w_e t_e c_j - D_i a_i) / tau     row kernel, over the CSR
//   dc_j = g_u,j + sum_{e=(i,j)} [w_e g_u,i + w_e (t_e - D_i) q_i / tau]            column kernel, over the transpose
// The row kernel accumulates sum w t c_j, a and D in one walk (a row with one edge gets exactly dq = 0) and writes
// g_u [n, F] and D [n, K] for the column kernel.  Both recompute s_e, t_e and w_e = 2^(z_e - lse2_i) from gathered
// rows with the same lane order, so t_e - D_i is exactly 0 where the forward's softmax had one term.  Hub rows /
// columns go through the plan of the CSR / the transpose, merged in chunk order.
//
// A zero-norm channel (|u| = 0) gives NaN, as the reference's division does: no epsilon (DESIGN 3.8).
#include "common.cuh"

#include <math_constants.h>

#include <cfloat>

namespace cogdl_b200 {

constexpr float DR_LOG2E = 1.4426950408889634f;

template <int W> struct DrVec;
template <> struct DrVec<1> { using T = float; };
template <> struct DrVec<4> { using T = float4; };

__device__ __forceinline__ void dr_unpack(const float &v, float (&o)[1]) { o[0] = v; }
__device__ __forceinline__ void dr_unpack(const float4 &v, float (&o)[4]) { o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; }
__device__ __forceinline__ float dr_pack(const float (&o)[1]) { return o[0]; }
__device__ __forceinline__ float4 dr_pack(const float (&o)[4]) { return make_float4(o[0], o[1], o[2], o[3]); }

template <int W>
__device__ __forceinline__ void dr_load(const float *base, int64_t off, bool ok, float (&o)[W]) {
  using VecT = typename DrVec<W>::T;
  if (ok) {
    dr_unpack(ld_gather(reinterpret_cast<const VecT *>(base) + off), o);
  } else {
#pragma unroll
    for (int k = 0; k < W; ++k) o[k] = 0.f;
  }
}

template <int W>
__device__ __forceinline__ float dr_dot(const float (&a)[W], const float (&b)[W]) {
  float s = a[0] * b[0];
#pragma unroll
  for (int k = 1; k < W; ++k) s = fmaf(a[k], b[k], s);
  return s;
}

// Sum over the L lanes of a channel (L a power of two, groups aligned).  The xor butterfly adds the same pairs in
// every lane, so all L lanes hold the same bits.
__device__ __forceinline__ float chan_sum(float v, int L, unsigned mask) {
  for (int o = L >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o);
  return v;
}
__device__ __forceinline__ void chan_sum2(float &a, float &b, int L, unsigned mask) {
  for (int o = L >> 1; o > 0; o >>= 1) {
    const float ta = __shfl_xor_sync(mask, a, o), tb = __shfl_xor_sync(mask, b, o);
    a += ta;
    b += tb;
  }
}

template <int GROUP>
__device__ __forceinline__ unsigned group_mask(int lane) {
  return GROUP == 32 ? FULL : (((1u << GROUP) - 1u) << (lane & ~(GROUP - 1)));
}

// gathers in flight per lane
template <int W, int GROUP> constexpr int dr_unroll() { return (W == 4 ? 4 : 8) < GROUP ? (W == 4 ? 4 : 8) : GROUP; }

struct DrFwdParams {
  const int *rowptr;
  const int *colind;
  const float *q;      // [n, F]
  const float *c;      // [n, F]
  float *out;          // [n, F]
  float *lse2;         // [n, K] or null (inference)
  float *r;            // [n, K] or null
  int64_t n_rows;
  int FV;              // row length in vectors
  int K;
  int L;               // lanes per channel, d / W
  int lgL;
  float zs;            // log2(e) / tau
  float *ms;           // hub partials (M, S) [n_chunks][K][2], after the acc partials [n_chunks][FV] vectors
  HubView hub;
};

// u = acc / S + c_i (u = c_i without edges), out = u / |u|; lse2 and r for the backward.  Called by every lane of
// the GROUP.  `any` comes from the CSR, not from S: a NaN channel of c (zero norm) makes S NaN in every row that
// routes to it, and the output must be NaN there, as the reference's softmax gives.
template <int W>
__device__ __forceinline__ void dr_fwd_finish(const DrFwdParams &p, int row, int cv, bool ok, bool any, float M,
                                              float S, const float (&acc)[W], unsigned mask) {
  using VecT = typename DrVec<W>::T;
  float u[W];
  dr_load<W>(p.c, (int64_t)row * p.FV + cv, ok, u);
  // a +Inf logit is its channel's max, and exp(z - max) = exp(Inf - Inf) is NaN in the softmax this restates: the
  // online state counted it as 1, so S is replaced by NaN here.  All logits -inf: S = 0, and acc / S is NaN.
  S = M < CUDART_INF_F ? S : CUDART_NAN_F;
#pragma unroll
  for (int k = 0; k < W; ++k) u[k] = any ? u[k] + acc[k] / S : u[k];
  const float nrm = sqrtf(chan_sum(dr_dot<W>(u, u), p.L, mask));
#pragma unroll
  for (int k = 0; k < W; ++k) u[k] = u[k] / nrm;
  if (!ok) return;
  st_stream(reinterpret_cast<VecT *>(p.out) + (int64_t)row * p.FV + cv, dr_pack(u));
  if (p.lse2 && (cv & (p.L - 1)) == 0) {
    const int64_t o = (int64_t)row * p.K + (cv >> p.lgL);
    p.lse2[o] = any ? M + log2f(S) : 0.f;
    p.r[o] = nrm;
  }
}

template <int W, int GROUP>
__global__ void __launch_bounds__(256) disen_route_fwd_kernel(const DrFwdParams p) {
  using VecT = typename DrVec<W>::T;
  constexpr int U = dr_unroll<W, GROUP>();
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const unsigned gmask = group_mask<GROUP>(lane);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const WorkItem w = decode_item(tid / GROUP, p.n_rows, p.rowptr, p.hub);
  const bool warp_has_chunk = (tid - lane) / GROUP < p.hub.n_chunks;   // warp-uniform
  const VecT *C = reinterpret_cast<const VecT *>(p.c);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  const int FV = p.FV;

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);   // warp-uniform trip counts: every lane joins the shuffles

  for (int tile0 = 0; tile0 < FV; tile0 += GROUP) {
    const int cv = tile0 + gl;
    const bool ok = w.active && cv < FV;
    float qi[W], acc[W];
    dr_load<W>(p.q, (int64_t)w.row * FV + cv, ok, qi);
#pragma unroll
    for (int k = 0; k < W; ++k) acc[k] = 0.f;
    // M starts at -FLT_MAX, not -inf: a -inf logit (a large q against its c) then gives e = 0 wherever it falls, where
    // -inf - (-inf) would make the channel NaN
    float M = -FLT_MAX, S = 0.f;
    for (int off = 0; off < maxdeg; off += GROUP) {
      const int cnt = min(GROUP, w.hb - w.lb - off);   // <= 0 once this item's edges are done
      const int cidx = gl < cnt ? ld_stream(p.colind + w.lb + off + gl) : 0;
#pragma unroll 1
      for (int j = 0; j < GROUP; j += U) {
        if (GROUP == 32) {
          if (j >= cnt) break;
        } else {
          if (!__any_sync(FULL, j < cnt)) break;
        }
        VecT xv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, cidx, j + u, GROUP);
          xv[u] = (ok && j + u < cnt) ? ld_gather(C + (int64_t)cj * FV + cv) : vzero<VecT>();
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float x[W];
          dr_unpack(xv[u], x);
          const float z = __fmul_rn(chan_sum(dr_dot<W>(qi, x), p.L, FULL), p.zs);
          if (ok && j + u < cnt) {
            const float dd = z - M;                 // first edge (z > -FLT_MAX): dd > 0, e = 0, S = 1, acc = x
            const float e = exp2f(-fabsf(dd));
            if (dd > 0.f) {
              S = fmaf(S, e, 1.f);
#pragma unroll
              for (int k = 0; k < W; ++k) acc[k] = fmaf(acc[k], e, x[k]);
              M = z;
            } else {
              S += e;
#pragma unroll
              for (int k = 0; k < W; ++k) acc[k] = fmaf(e, x[k], acc[k]);
            }
          }
        }
      }
    }
    if (w.is_chunk) {
      if (ok) {
        st_cg(P + (int64_t)w.slot * FV + cv, dr_pack(acc));
        if ((cv & (p.L - 1)) == 0) {
          float *m = p.ms + ((int64_t)w.slot * p.K + (cv >> p.lgL)) * 2;
          st_cg(m, M);
          st_cg(m + 1, S);
        }
      }
    } else if (w.active) {
      dr_fwd_finish<W>(p, w.row, cv, ok, w.hb > w.lb, M, S, acc, gmask);
    }
  }

  if (warp_has_chunk && hub_arrive_last<GROUP>(w, p.hub, gl)) {
    for (int tile0 = 0; tile0 < FV; tile0 += GROUP) {
      const int cv = tile0 + gl;
      const bool ok = cv < FV;
      const int64_t mo = (cv >> p.lgL) * 2;
      struct Part { float M, S, a[W]; };
      const Part s = merge_chunks<1>(
          w.n_row_chunks,
          [&](int qq) {
            Part t;
            t.M = 0.f;
            t.S = 1.f;
#pragma unroll
            for (int k = 0; k < W; ++k) t.a[k] = 0.f;
            if (ok) {
              const int64_t slot = w.first + qq;
              dr_unpack(ld_cg(P + slot * FV + cv), t.a);
              t.M = ld_cg(p.ms + slot * p.K * 2 + mo);
              t.S = ld_cg(p.ms + slot * p.K * 2 + mo + 1);
            }
            return t;
          },
          [](Part &a, const Part &t) {   // every chunk has an edge
            const float Mn = fmaxf(a.M, t.M);
            const float ea = exp2f(a.M - Mn), eb = exp2f(t.M - Mn);
            a.S = fmaf(a.S, ea, t.S * eb);
#pragma unroll
            for (int k = 0; k < W; ++k) a.a[k] = fmaf(a.a[k], ea, t.a[k] * eb);
            a.M = Mn;
          });
      dr_fwd_finish<W>(p, w.row, cv, ok, true, s.M, s.S, s.a, gmask);
    }
  }
}

struct DrRowBwdParams {
  const int *rowptr;
  const int *colind;
  const float *q, *c, *g, *out;   // [n, F]
  const float *lse2, *r;          // [n, K]
  float *gu;                      // [n, F] out
  float *D;                       // [n, K] out
  float *dq;                      // [n, F] out
  int64_t n_rows;
  int FV, K, L, lgL;
  float zs, tau;
  float *pa, *pd;                 // hub partials: A1 [n_chunks][FV] vectors (hub.partials), A2 (pa), D [n_chunks][K] (pd)
  HubView hub;                    // CSR plan
};

// dq = (A1 - D A2) / tau with A1 = sum_e w t c_j, A2 = sum_e w c_j (= a), D = sum_e w t (= g_u . a), t = g_u . c_j.
// All three come from one walk, so a row with one edge (w = 1) gives exactly 0, as the softmax backward must.
template <int W>
__device__ __forceinline__ void dr_row_finish(const DrRowBwdParams &p, int row, int cv, const float (&a1)[W],
                                              const float (&a2)[W], float D) {
  using VecT = typename DrVec<W>::T;
  float o[W];
#pragma unroll
  for (int k = 0; k < W; ++k) o[k] = __fsub_rn(a1[k], __fmul_rn(D, a2[k])) / p.tau;
  st_stream(reinterpret_cast<VecT *>(p.dq) + (int64_t)row * p.FV + cv, dr_pack(o));
  if ((cv & (p.L - 1)) == 0) p.D[(int64_t)row * p.K + (cv >> p.lgL)] = D;
}

template <int W, int GROUP>
__global__ void __launch_bounds__(256) disen_route_bwd_row_kernel(const DrRowBwdParams p) {
  using VecT = typename DrVec<W>::T;
  constexpr int U = dr_unroll<W, GROUP>();
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const WorkItem w = decode_item(tid / GROUP, p.n_rows, p.rowptr, p.hub);
  const bool warp_has_chunk = (tid - lane) / GROUP < p.hub.n_chunks;
  const VecT *C = reinterpret_cast<const VecT *>(p.c);
  VecT *P1 = reinterpret_cast<VecT *>(p.hub.partials);
  VecT *P2 = reinterpret_cast<VecT *>(p.pa);
  const int FV = p.FV;

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);

  for (int tile0 = 0; tile0 < FV; tile0 += GROUP) {
    const int cv = tile0 + gl;
    const bool ok = w.active && cv < FV;
    const int64_t ro = (int64_t)w.row * FV + cv;
    const int64_t ko = (int64_t)w.row * p.K + (cv >> p.lgL);
    float qi[W], gi[W], oi[W], gu[W], a1[W], a2[W];
    dr_load<W>(p.q, ro, ok, qi);
    dr_load<W>(p.g, ro, ok, gi);
    dr_load<W>(p.out, ro, ok, oi);
    const float rr = ok ? __ldg(p.r + ko) : 1.f;
    const float lse = ok ? __ldg(p.lse2 + ko) : 0.f;
    const float og = chan_sum(dr_dot<W>(oi, gi), p.L, FULL);
#pragma unroll
    for (int k = 0; k < W; ++k) {
      gu[k] = (gi[k] - oi[k] * og) / rr;
      a1[k] = 0.f;
      a2[k] = 0.f;
    }
    float D = 0.f;
    if (ok && (!w.is_chunk || w.slot == w.first))   // every chunk computes g_u; one writes it
      st_stream(reinterpret_cast<VecT *>(p.gu) + ro, dr_pack(gu));
    for (int off = 0; off < maxdeg; off += GROUP) {
      const int cnt = min(GROUP, w.hb - w.lb - off);
      const int cidx = gl < cnt ? ld_stream(p.colind + w.lb + off + gl) : 0;
#pragma unroll 1
      for (int j = 0; j < GROUP; j += U) {
        if (GROUP == 32) {
          if (j >= cnt) break;
        } else {
          if (!__any_sync(FULL, j < cnt)) break;
        }
        VecT xv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, cidx, j + u, GROUP);
          xv[u] = (ok && j + u < cnt) ? ld_gather(C + (int64_t)cj * FV + cv) : vzero<VecT>();
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float x[W];
          dr_unpack(xv[u], x);
          float s = dr_dot<W>(qi, x), t = dr_dot<W>(gu, x);
          chan_sum2(s, t, p.L, FULL);
          if (ok && j + u < cnt) {
            const float wgt = exp2f(__fmul_rn(s, p.zs) - lse);
            const float wt = __fmul_rn(wgt, t);
            D = __fadd_rn(D, wt);
#pragma unroll
            for (int k = 0; k < W; ++k) {
              a1[k] = fmaf(wt, x[k], a1[k]);
              a2[k] = fmaf(wgt, x[k], a2[k]);
            }
          }
        }
      }
    }
    if (w.is_chunk) {
      if (ok) {
        st_cg(P1 + (int64_t)w.slot * FV + cv, dr_pack(a1));
        st_cg(P2 + (int64_t)w.slot * FV + cv, dr_pack(a2));
        if ((cv & (p.L - 1)) == 0) st_cg(p.pd + (int64_t)w.slot * p.K + (cv >> p.lgL), D);
      }
    } else if (ok) {
      dr_row_finish<W>(p, w.row, cv, a1, a2, D);
    }
  }

  if (warp_has_chunk && hub_arrive_last<GROUP>(w, p.hub, gl)) {
    for (int cv = gl; cv < FV; cv += GROUP) {
      struct Part { float a1[W], a2[W], D; };
      const Part s = merge_chunks<1>(
          w.n_row_chunks,
          [&](int qq) {
            const int64_t slot = w.first + qq;
            Part t;
            dr_unpack(ld_cg(P1 + slot * FV + cv), t.a1);
            dr_unpack(ld_cg(P2 + slot * FV + cv), t.a2);
            t.D = ld_cg(p.pd + slot * p.K + (cv >> p.lgL));
            return t;
          },
          [](Part &a, const Part &t) {
#pragma unroll
            for (int k = 0; k < W; ++k) {
              a.a1[k] = __fadd_rn(a.a1[k], t.a1[k]);
              a.a2[k] = __fadd_rn(a.a2[k], t.a2[k]);
            }
            a.D = __fadd_rn(a.D, t.D);
          });
      dr_row_finish<W>(p, w.row, cv, s.a1, s.a2, s.D);
    }
  }
}

struct DrColBwdParams {
  const int *colptr;
  const int *rowind;
  const float *q, *c, *gu;     // [n, F]
  const float *lse2, *D;       // [n, K]
  float *dc;                   // [n, F] out
  int64_t n_cols;
  int FV, K, L, lgL;
  float zs, tau;
  HubView hub;                 // the transpose's plan; partials [n_chunks][FV] vectors
};

template <int W, int GROUP>
__global__ void __launch_bounds__(256) disen_route_bwd_col_kernel(const DrColBwdParams p) {
  using VecT = typename DrVec<W>::T;
  constexpr int U = dr_unroll<W, GROUP>();
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const WorkItem w = decode_item(tid / GROUP, p.n_cols, p.colptr, p.hub);
  const bool warp_has_chunk = (tid - lane) / GROUP < p.hub.n_chunks;
  const VecT *Qv = reinterpret_cast<const VecT *>(p.q);
  const VecT *GU = reinterpret_cast<const VecT *>(p.gu);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  VecT *DC = reinterpret_cast<VecT *>(p.dc);
  const int FV = p.FV;

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);

  for (int tile0 = 0; tile0 < FV; tile0 += GROUP) {
    const int cv = tile0 + gl;
    const bool ok = w.active && cv < FV;
    const int kc = cv >> p.lgL;
    float cj[W], acc[W];
    dr_load<W>(p.c, (int64_t)w.row * FV + cv, ok, cj);
#pragma unroll
    for (int k = 0; k < W; ++k) acc[k] = 0.f;
    for (int off = 0; off < maxdeg; off += GROUP) {
      const int cnt = min(GROUP, w.hb - w.lb - off);
      const int ridx = gl < cnt ? ld_stream(p.rowind + w.lb + off + gl) : 0;
#pragma unroll 1
      for (int j = 0; j < GROUP; j += U) {
        if (GROUP == 32) {
          if (j >= cnt) break;
        } else {
          if (!__any_sync(FULL, j < cnt)) break;
        }
        VecT qv[U], gv[U];
        float lv[U], dv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int ri = __shfl_sync(FULL, ridx, j + u, GROUP);
          const bool live = ok && j + u < cnt;
          const int64_t ro = (int64_t)ri * FV + cv, ko = (int64_t)ri * p.K + kc;
          qv[u] = live ? ld_gather(Qv + ro) : vzero<VecT>();
          gv[u] = live ? ld_gather(GU + ro) : vzero<VecT>();
          lv[u] = live ? __ldg(p.lse2 + ko) : 0.f;
          dv[u] = live ? __ldg(p.D + ko) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float qf[W], gf[W];
          dr_unpack(qv[u], qf);
          dr_unpack(gv[u], gf);
          float s = dr_dot<W>(qf, cj), t = dr_dot<W>(gf, cj);
          chan_sum2(s, t, p.L, FULL);
          if (ok && j + u < cnt) {
            const float wgt = exp2f(__fmul_rn(s, p.zs) - lv[u]);
            const float coef = wgt * (t - dv[u]) / p.tau;
#pragma unroll
            for (int k = 0; k < W; ++k) acc[k] = fmaf(wgt, gf[k], fmaf(coef, qf[k], acc[k]));
          }
        }
      }
    }
    if (w.is_chunk) {
      if (ok) st_cg(P + (int64_t)w.slot * FV + cv, dr_pack(acc));
    } else if (ok) {
      float gj[W];
      dr_unpack(ld_gather(GU + (int64_t)w.row * FV + cv), gj);
#pragma unroll
      for (int k = 0; k < W; ++k) acc[k] = gj[k] + acc[k];   // the residual u = a + c
      st_stream(DC + (int64_t)w.row * FV + cv, dr_pack(acc));
    }
  }

  if (warp_has_chunk && hub_arrive_last<GROUP>(w, p.hub, gl)) {
    for (int cv = gl; cv < FV; cv += GROUP) {
      const VecT *pp = P + (int64_t)w.first * FV + cv;
      const VecT s = merge_chunks<1>(w.n_row_chunks, [&](int qq) { return ld_cg(pp + (int64_t)qq * FV); },
                                     [](VecT &a, const VecT &t) { add_rn(a, t); });
      float o[W], gj[W];
      dr_unpack(s, o);
      dr_unpack(ld_gather(GU + (int64_t)w.row * FV + cv), gj);
#pragma unroll
      for (int k = 0; k < W; ++k) o[k] = gj[k] + o[k];
      st_stream(DC + (int64_t)w.row * FV + cv, dr_pack(o));
    }
  }
}

// Lanes per row: the smallest power of two covering the row's vectors, at most a warp (wider rows loop over tiles).
static int dr_group(int FV) {
  int g = 1;
  while (g < FV && g < 32) g <<= 1;
  return g;
}

static int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

#define DR_KERNEL_TABLE(NAME, PARAMS)                                                                        \
  template <int W>                                                                                           \
  static int launch_##NAME(const PARAMS &p, int64_t items, int group, cudaStream_t s, const char *who) {     \
    const char *fmt = "cogdl_b200::" #NAME "_kernel<%s,GROUP=%d>";                                        \
    const char *vt = W == 4 ? "float4" : "float";                                                             \
    switch (group) {                                                                                          \
      case 1: return launch_items(NAME##_kernel<W, 1>, p, items, 1, s, who, fmt, vt, 1);                      \
      case 2: return launch_items(NAME##_kernel<W, 2>, p, items, 2, s, who, fmt, vt, 2);                      \
      case 4: return launch_items(NAME##_kernel<W, 4>, p, items, 4, s, who, fmt, vt, 4);                      \
      case 8: return launch_items(NAME##_kernel<W, 8>, p, items, 8, s, who, fmt, vt, 8);                      \
      case 16: return launch_items(NAME##_kernel<W, 16>, p, items, 16, s, who, fmt, vt, 16);                  \
      default: return launch_items(NAME##_kernel<W, 32>, p, items, 32, s, who, fmt, vt, 32);                  \
    }                                                                                                         \
  }

DR_KERNEL_TABLE(disen_route_fwd, DrFwdParams)
DR_KERNEL_TABLE(disen_route_bwd_row, DrRowBwdParams)
DR_KERNEL_TABLE(disen_route_bwd_col, DrColBwdParams)
#undef DR_KERNEL_TABLE

// Shape checks shared by both directions; sets *d.
static int dr_check_shape(const char *who, int64_t n_rows, int64_t n_cols, int64_t F, int64_t K, float tau,
                          int64_t *d) {
  CB_REQUIRE(n_rows >= 0 && n_cols >= 0 && F >= 0, "%s: negative size", who);
  CB_REQUIRE(n_rows == n_cols, "%s: the routing needs a square structure (n_rows=%lld, n_cols=%lld)", who,
             (long long)n_rows, (long long)n_cols);
  CB_REQUIRE(K >= 1 && F % K == 0, "%s: F=%lld is not a multiple of K=%lld channels", who, (long long)F, (long long)K);
  *d = F / K;
  CB_REQUIRE(*d >= 1 && *d <= 32 && (*d & (*d - 1)) == 0,
             "%s: channel width d=%lld is not supported (powers of two from 1 to 32)", who, (long long)*d);
  CB_REQUIRE(tau > 0.f && tau <= FLT_MAX,"%s: tau must be positive and finite, got %g", who, (double)tau);
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "%s: sizes must fit int32", who);
  return COGDL_B200_OK;
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_disen_route_scratch_bytes(int64_t n_chunks, int64_t F, int64_t K) {
  return n_chunks > 0 && F > 0 && K > 0 ? n_chunks * (2 * F + 2 * K) * 4 : 0;
}

extern "C" int cogdl_b200_disen_route_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *q,
                                              const float *c, float *out, float *lse2, float *r, int64_t n_rows,
                                              int64_t n_cols, int64_t F, int64_t K, float tau,
                                              const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_disen_route_fwd_f32";
  int64_t d = 0;
  int rc = dr_check_shape(who, n_rows, n_cols, F, K, tau, &d);
  if (rc) return rc;
  if (n_rows == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && q && c && out, "%s: null pointer", who);
  CB_REQUIRE((lse2 == nullptr) == (r == nullptr), "%s: lse2 and r are written together", who);
  const int64_t n_chunks = plan && plan->chunk_edges > 0 ? plan->n_chunks : 0;
  rc = check_plan(plan, cogdl_b200_disen_route_scratch_bytes(n_chunks, F, K));
  if (rc) return rc;
  DrFwdParams p;
  p.rowptr = rowptr; p.colind = colind; p.q = q; p.c = c; p.out = out; p.lse2 = lse2; p.r = r;
  p.n_rows = n_rows; p.K = (int)K; p.zs = DR_LOG2E / tau;
  p.hub = hub_view(plan);
  p.ms = n_chunks > 0 ? reinterpret_cast<float *>(p.hub.partials) + n_chunks * F : nullptr;
  const bool vec = d % 4 == 0 && aligned16(q) && aligned16(c) && aligned16(out) &&
                   (n_chunks == 0 || aligned16(p.hub.partials));
  const int W = vec ? 4 : 1;
  p.FV = (int)(F / W);
  p.L = (int)(d / W);
  p.lgL = ilog2(p.L);
  const int64_t items = n_chunks + n_rows;
  cudaStream_t s = (cudaStream_t)stream;
  return vec ? launch_disen_route_fwd<4>(p, items, dr_group(p.FV), s, who)
             : launch_disen_route_fwd<1>(p, items, dr_group(p.FV), s, who);
}

extern "C" int cogdl_b200_disen_route_bwd_f32(const int32_t *rowptr, const int32_t *colind,
                                              const cogdl_b200_hub_plan_t *plan, const int32_t *colptr,
                                              const int32_t *rowind, const cogdl_b200_hub_plan_t *plan_t,
                                              const float *q, const float *c, const float *G, const float *out,
                                              const float *lse2, const float *r, float *g_u, float *D, float *dq,
                                              float *dc, int64_t n_rows, int64_t n_cols, int64_t F, int64_t K,
                                              float tau, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_disen_route_bwd_f32";
  int64_t d = 0;
  int rc = dr_check_shape(who, n_rows, n_cols, F, K, tau, &d);
  if (rc) return rc;
  if (n_rows == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && colptr && rowind && q && c && G && out && lse2 && r && g_u && D && dq && dc,
             "%s: null pointer", who);
  const int64_t n_chunks = plan && plan->chunk_edges > 0 ? plan->n_chunks : 0;
  const int64_t n_chunks_t = plan_t && plan_t->chunk_edges > 0 ? plan_t->n_chunks : 0;
  rc = check_plan(plan, cogdl_b200_disen_route_scratch_bytes(n_chunks, F, K));
  if (rc) return rc;
  rc = check_plan(plan_t, cogdl_b200_disen_route_scratch_bytes(n_chunks_t, F, K));
  if (rc) return rc;
  const bool vec = d % 4 == 0 && aligned16(q) && aligned16(c) && aligned16(G) && aligned16(out) && aligned16(g_u) &&
                   aligned16(dq) && aligned16(dc) && (n_chunks == 0 || aligned16(plan->partials)) &&
                   (n_chunks_t == 0 || aligned16(plan_t->partials));
  const int W = vec ? 4 : 1;
  const int FV = (int)(F / W), L = (int)(d / W), lgL = ilog2(L), group = dr_group(FV);
  const float zs = DR_LOG2E / tau;
  cudaStream_t s = (cudaStream_t)stream;

  DrRowBwdParams pr;
  pr.rowptr = rowptr; pr.colind = colind; pr.q = q; pr.c = c; pr.g = G; pr.out = out; pr.lse2 = lse2; pr.r = r;
  pr.gu = g_u; pr.D = D; pr.dq = dq; pr.n_rows = n_rows;
  pr.FV = FV; pr.K = (int)K; pr.L = L; pr.lgL = lgL; pr.zs = zs; pr.tau = tau;
  pr.hub = hub_view(plan);
  pr.pa = n_chunks > 0 ? reinterpret_cast<float *>(pr.hub.partials) + n_chunks * F : nullptr;
  pr.pd = n_chunks > 0 ? pr.pa + n_chunks * F : nullptr;
  rc = vec ? launch_disen_route_bwd_row<4>(pr, n_chunks + n_rows, group, s, who)
           : launch_disen_route_bwd_row<1>(pr, n_chunks + n_rows, group, s, who);
  if (rc) return rc;

  DrColBwdParams pc;
  pc.colptr = colptr; pc.rowind = rowind; pc.q = q; pc.c = c; pc.gu = g_u; pc.lse2 = lse2; pc.D = D; pc.dc = dc;
  pc.n_cols = n_cols; pc.FV = FV; pc.K = (int)K; pc.L = L; pc.lgL = lgL; pc.zs = zs; pc.tau = tau;
  pc.hub = hub_view(plan_t);
  rc = vec ? launch_disen_route_bwd_col<4>(pc, n_chunks_t + n_cols, group, s, who)
           : launch_disen_route_bwd_col<1>(pc, n_chunks_t + n_cols, group, s, who);
  if (rc) return rc;
  note_kernel("cogdl_b200::disen_route_bwd_row_kernel<%s,GROUP=%d> + cogdl_b200::disen_route_bwd_col_kernel<%s,GROUP=%d>",
              vec ? "float4" : "float", group, vec ? "float4" : "float", group);
  return COGDL_B200_OK;
}

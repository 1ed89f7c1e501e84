// edge_softmax.cuh -- the per-row softmax kernels of edge_softmax.cu (MODES 0-3, see its header comment) and their
// launch plan, es_launch.  simple_hgn.cu launches the attention forms with two more flags:
//   TYPED (MODES 2, 3): the logit gains a per-edge-type term, leakyrelu(h_l[row,h] + h_r[col,h] + h_e[type[p],h]),
//          h_e [T, H] staged in shared memory by the kernel (`tab`), type [nnz] int32 in CSR slot order;
//   MIX   (MODE 2, TYPED only): besides the signed softmax (out, nullable), the kernel writes the attention the layer
//          returns, mix = (1 - alpha) * a * (dropped ? 0 : keep_scale) + alpha * res[p,h]; without MIX it is
//          a * (dropped ? 0 : keep_scale), a product, so a dropped NaN stays NaN.
// edge_softmax.cu launches them with TYPED = MIX = false.
#pragma once
#include "common.cuh"
#include "rng.cuh"

#include <math_constants.h>

#include <cfloat>
#include <cstdio>
#include <cstdlib>

namespace cogdl_b200 {

struct EsParams {
  const int *rowptr;
  const float *a;
  const float *b;
  float *out;
  int64_t n_rows;
  int H;
  int lgH;
  const int *colind = nullptr;  // MODE 2, 3
  float slope = 0.f;            // MODE 2, 3
  const float *hl = nullptr;    // MODE 3: h_l [N,H]
  const float *hr = nullptr;    // MODE 3: h_r [N,H]
  float *grow = nullptr;        // MODE 3: [N,H] row sums of the output
  HubView hub;            // chunks / segments / edge_row / counters
  float2 *stats;          // per chunk slot x head: (max, sum) -- the row's merged value sits in its first slot
  float *part;            // MODE 3: per chunk slot x head partial row sums
  bool bulk;              // tiles may be moved with cp.async.bulk (alignment checked on the host)
  uint64_t seed = 0;            // DROP: attention-dropout mask (see the header comment of edge_softmax.cu)
  uint64_t drop_below = 0;
  float scale = 1.f;            // DROP, MODE 3: the factor d att is multiplied by on a kept entry
  // TYPED / MIX (simple_hgn.cu)
  const int *etype = nullptr;   // TYPED: edge type of each CSR slot, in [0, T)
  const float *he = nullptr;    // TYPED: h_e [T, H], copied to `tab` by the kernel
  int n_table = 0;              // TYPED: T * H
  float *mix = nullptr;         // TYPED, MODE 2: the returned attention [nnz, H]; `out` (the signed softmax) may be null
  const float *res = nullptr;   // MIX: res_attn [nnz, H]
  float alpha = 0.f;            // MIX: weight of res_attn
  float keep = 1.f;             // MIX: 1 - alpha
  float keep_scale = 1.f;       // TYPED, MODE 2: factor of a kept attention in mix (1 / (1 - p_drop))
};

// DROP, MODE 2: the attention a (>= 0) of CSR edge `edge`, head `head`, with the sign bit set if the pair is dropped
template <bool DROP>
__device__ __forceinline__ float es_mark(const EsParams &p, int64_t edge, int head, float a) {
  if (DROP && draw(p.seed, edge, head) < p.drop_below) a = __uint_as_float(__float_as_uint(a) | 0x80000000u);
  return a;
}
// DROP, MODE 3: (y, g) = (saved attention, d attention after dropout) -> (softmax, d softmax)
template <bool DROP>
__device__ __forceinline__ void es_unmark(const EsParams &p, float &y, float &g) {
  if (DROP) {
    // a product with 0, not a select: a NaN or Inf gradient of a dropped entry gives NaN, as torch's g * mask * scale
    g = __fmul_rn(g, __int_as_float(~(__float_as_int(y) >> 31) & __float_as_int(p.scale)));
    y = fabsf(y);
  }
}

// MODE 2: store the (signed) attention a of element k of the [nnz, H] output.  TYPED: also the returned attention.
template <bool TYPED, bool MIX>
__device__ __forceinline__ void es_put(const EsParams &p, int64_t k, float a) {
  if (!TYPED) {
    st_stream(p.out + k, a);
    return;
  }
  if (p.out) st_stream(p.out + k, a);
  // |a| * (kept ? keep_scale : 0), a product and not a select: a dropped NaN stays NaN
  float m = __fmul_rn(fabsf(a), __int_as_float(~(__float_as_int(a) >> 31) & __float_as_int(p.keep_scale)));
  if (MIX) m = __fadd_rn(__fmul_rn(m, p.keep), __fmul_rn(__ldg(p.res + k), p.alpha));
  st_stream(p.mix + k, m);
}

// TYPED: add the type term of CSR edge e, head h to the pre-activation z (h_l + h_r, in the reference's order)
template <bool TYPED>
__device__ __forceinline__ float es_typed(const EsParams &p, const float *tab, int64_t e, int head, float z) {
  if (TYPED) z += tab[__ldg(p.etype + e) * p.H + head];
  return z;
}

constexpr int HGN_MAX_TABLE = 1024;   // the largest T * H: the floats of a kernel's static shared table for h_e

// TAB (the kernel reads the type term): copy h_e into the block's table, declared table[TAB ? HGN_MAX_TABLE : 1], and
// return it; else return null.  Every thread of the block calls this before any early exit.
template <bool TAB>
__device__ __forceinline__ const float *es_stage_table(const EsParams &p, float *table) {
  if (TAB) {
    for (int i = threadIdx.x; i < p.n_table; i += blockDim.x) table[i] = __ldg(p.he + i);
    __syncthreads();
  }
  return TAB ? table : nullptr;
}

// exp for the plan-based kernels: arguments are x - max <= 0.  ex2.approx(x * log2 e): 2 ulp from the MUFU plus
// |x| * 2^-24 from the scaling product, i.e. <= ~2e-6 relative for logits within 30 of the row maximum and an
// absolute error far below 1e-5 of the row's largest term beyond that (parity bar: 1e-5).  FMUL + MUFU.EX2
// instead of the ~12-instruction expf(): these kernels are issue-bound, not memory-bound.
__device__ __forceinline__ float es_exp(float x) { return __expf(x); }

// reduce across lanes that share lane % H  (strides 16 .. H)
__device__ __forceinline__ float head_max(float v, int H) {
  for (int s = 16; s >= H; s >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, s));
  return v;
}
__device__ __forceinline__ float head_sum(float v, int H) {
  for (int s = 16; s >= H; s >>= 1) v += __shfl_xor_sync(FULL, v, s);
  return v;
}

// Forward input of element t of the row whose block starts at edge lb (head = t % H).
template <int MODE, bool TYPED>
__device__ __forceinline__ float es_in(const EsParams &p, const float *tab, int lb, int64_t t, int head, float hl) {
  if (MODE == 2) {
    const int e = lb + (int)(t >> p.lgH);
    const int c = __ldg(p.colind + e);
    const float z = es_typed<TYPED>(p, tab, e, head, hl + __ldg(p.b + (int64_t)c * p.H + head));
    return z > 0.f ? z : z * p.slope;
  }
  return __ldg(p.a + (int64_t)lb * p.H + t);
}
// MODE 3: derivative of the LeakyReLU at the pre-activation of element t
template <bool TYPED>
__device__ __forceinline__ float es_dact(const EsParams &p, const float *tab, int lb, int64_t t, int head, float hlrow) {
  const int e = lb + (int)(t >> p.lgH);
  const int c = __ldg(p.colind + e);
  const float z = es_typed<TYPED>(p, tab, e, head, hlrow + __ldg(p.hr + (int64_t)c * p.H + head));
  return z > 0.f ? 1.f : p.slope;
}

// One row handled by a team of NT threads striding the row's elements (tid = index inside the
// team, NT % H == 0).  reduce(v, is_max) must return the team-wide per-head reduction.
template <int MODE, int NT, bool DROP, bool TYPED, bool MIX, typename Reduce>
__device__ __forceinline__ void es_row(const EsParams &p, const float *tab, int64_t row, int lb, int64_t n, int tid,
                                       Reduce reduce) {
  const int head = tid & (p.H - 1);
  float *o = p.out + (int64_t)lb * p.H;
  const int64_t ob = (int64_t)lb * p.H;
  if (MODE == 1 || MODE == 3) {
    const float *y = p.a + (int64_t)lb * p.H, *g = p.b + (int64_t)lb * p.H;
    auto yg = [&](int64_t t) {
      float yv = __ldg(y + t), gv = __ldg(g + t);
      es_unmark<DROP>(p, yv, gv);
      return make_float2(yv, gv);
    };
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int64_t t = tid;
    for (; t + 3 * NT < n; t += 4 * NT) {
      float2 v = yg(t);
      s0 = fmaf(v.x, v.y, s0);
      v = yg(t + NT);
      s1 = fmaf(v.x, v.y, s1);
      v = yg(t + 2 * NT);
      s2 = fmaf(v.x, v.y, s2);
      v = yg(t + 3 * NT);
      s3 = fmaf(v.x, v.y, s3);
    }
    for (; t < n; t += NT) { const float2 v = yg(t); s0 = fmaf(v.x, v.y, s0); }
    const float s = reduce((s0 + s1) + (s2 + s3), false);
    t = tid;
    if (MODE == 1) {
#pragma unroll 4
      for (; t < n; t += NT) st_stream(o + t, __ldg(y + t) * (__ldg(g + t) - s));
    } else {
      const float hlrow = __ldg(p.hl + row * p.H + head);
      float acc = 0.f;
      for (; t < n; t += NT) {
        const float2 w = yg(t);
        const float v = w.x * (w.y - s) * es_dact<TYPED>(p, tab, lb, t, head, hlrow);
        st_stream(o + t, v);
        acc += v;
      }
      acc = reduce(acc, false);
      if (tid < p.H) p.grow[row * p.H + head] = acc;
    }
    return;
  }
  const float hl = (MODE == 2) ? __ldg(p.a + row * p.H + head) : 0.f;
  auto in = [&](int64_t t) { return es_in<MODE, TYPED>(p, tab, lb, t, head, hl); };
  float m0 = -CUDART_INF_F, m1 = m0, m2 = m0, m3 = m0;
  int64_t t = tid;
  for (; t + 3 * NT < n; t += 4 * NT) {
    const float x0 = in(t), x1 = in(t + NT), x2 = in(t + 2 * NT), x3 = in(t + 3 * NT);
    m0 = fmaxf(m0, x0); m1 = fmaxf(m1, x1); m2 = fmaxf(m2, x2); m3 = fmaxf(m3, x3);
  }
  for (; t < n; t += NT) m0 = fmaxf(m0, in(t));
  const float m = reduce(fmaxf(fmaxf(m0, m1), fmaxf(m2, m3)), true);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  t = tid;
  for (; t + 3 * NT < n; t += 4 * NT) {
    const float x0 = in(t), x1 = in(t + NT), x2 = in(t + 2 * NT), x3 = in(t + 3 * NT);
    s0 += expf(x0 - m); s1 += expf(x1 - m); s2 += expf(x2 - m); s3 += expf(x3 - m);
  }
  for (; t < n; t += NT) s0 += expf(in(t) - m);
  const float s = reduce((s0 + s1) + (s2 + s3), false);
  t = tid;
  for (; t + 3 * NT < n; t += 4 * NT) {
    const float x0 = in(t), x1 = in(t + NT), x2 = in(t + 2 * NT), x3 = in(t + 3 * NT);
    const int64_t e = lb + (t >> p.lgH), de = NT >> p.lgH;     // CSR edge of element t (DROP)
    es_put<TYPED, MIX>(p, ob + t, es_mark<DROP>(p, e, head, expf(x0 - m) / s));
    es_put<TYPED, MIX>(p, ob + t + NT, es_mark<DROP>(p, e + de, head, expf(x1 - m) / s));
    es_put<TYPED, MIX>(p, ob + t + 2 * NT, es_mark<DROP>(p, e + 2 * de, head, expf(x2 - m) / s));
    es_put<TYPED, MIX>(p, ob + t + 3 * NT, es_mark<DROP>(p, e + 3 * de, head, expf(x3 - m) / s));
  }
  for (; t < n; t += NT) es_put<TYPED, MIX>(p, ob + t, es_mark<DROP>(p, lb + (t >> p.lgH), head, expf(in(t) - m) / s));
}

// ---------------------------------------------------------------- warp per row (no plan)
template <int MODE, bool DROP, bool TYPED, bool MIX>
__global__ void __launch_bounds__(256) es_warp_kernel(const EsParams p) {
  __shared__ float table[TYPED ? HGN_MAX_TABLE : 1];
  const float *tab = es_stage_table<TYPED>(p, table);
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= p.n_rows) return;  // whole warp
  const int lb = __ldg(p.rowptr + row), hb = __ldg(p.rowptr + row + 1);
  const int64_t n = (int64_t)(hb - lb) * p.H;
  const int H = p.H;
  if (n == 0) {
    if (MODE == 3 && lane < H) p.grow[row * H + lane] = 0.f;
    return;
  }
  es_row<MODE, 32, DROP, TYPED, MIX>(p, tab, row, lb, n, lane,
                                      [H](float v, bool is_max) { return is_max ? head_max(v, H) : head_sum(v, H); });
}

// ---------------------------------------------------------------- hub chunks, pass 1: statistics
// One warp per chunk slot.  Forward / attention: (max, sum exp(x - max)) per head; backward: sum y*g.
// The last chunk of the row to arrive merges the chunks' values in chunk order into stats[first].  A typed MODE 3
// sums a * g and forms no logit, so of the typed forms only MODE 2 reads the type table.
template <int MODE, bool DROP, bool TYPED>
__global__ void __launch_bounds__(256) es_stats_kernel(const EsParams p) {
  constexpr bool TAB = TYPED && MODE == 2;
  __shared__ float table[TAB ? HGN_MAX_TABLE : 1];
  const float *tab = es_stage_table<TAB>(p, table);
  // programmatic dependent launch: the main kernel may start as soon as every CTA of this grid is running; its
  // segment items need nothing from us, its chunk items wait (griddepcontrol.wait) for this grid to finish
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int lane = threadIdx.x & 31;
  const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (item >= p.hub.n_chunks) return;
  const WorkItem w = decode_item(item, 0, p.rowptr, p.hub);
  const int H = p.H, head = lane & (H - 1);
  const int n = (w.hb - w.lb) * H;
  float m = -CUDART_INF_F, s = 0.f;
  if (MODE == 1 || MODE == 3) {
    const float *y = p.a + (int64_t)w.lb * H, *g = p.b + (int64_t)w.lb * H;
    for (int t = lane; t < n; t += 32) {
      float yv = __ldg(y + t), gv = __ldg(g + t);
      es_unmark<DROP>(p, yv, gv);
      s = fmaf(yv, gv, s);
    }
    s = head_sum(s, H);
  } else {
    const float hl = (MODE == 2) ? __ldg(p.a + (int64_t)w.row * H + head) : 0.f;
    for (int t = lane; t < n; t += 32) m = fmaxf(m, es_in<MODE, TAB>(p, tab, w.lb, t, head, hl));
    m = head_max(m, H);
    for (int t = lane; t < n; t += 32) s += es_exp(es_in<MODE, TAB>(p, tab, w.lb, t, head, hl) - m);   // L1 hits
    s = head_sum(s, H);
  }
  if (lane < H) {
    float2 *dst = p.stats + (int64_t)w.slot * H + lane;
    asm volatile("st.global.cg.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(m), "f"(s) : "memory");
  }
  if (hub_arrive_last<32>(w, p.hub, lane)) {
    // lanes sharing a head split the chunks between them, then merge across the head's lanes
    const int grp = lane >> p.lgH, ngrp = 32 >> p.lgH;
    float M = -CUDART_INF_F, S = 0.f;
    const float2 *sb = p.stats + (int64_t)w.first * H + head;
    for (int q0 = grp; q0 < w.n_row_chunks; q0 += 4 * ngrp) {
      float2 c[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {        // four independent L2 loads in flight (the 22 K-edge hub merges 354 chunks)
        const int q = q0 + u * ngrp;
        c[u] = (q < w.n_row_chunks) ? __ldcg(sb + (int64_t)q * H) : make_float2(-CUDART_INF_F, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (MODE == 1 || MODE == 3) {
          S += c[u].y;
        } else if (c[u].x != -CUDART_INF_F) {
          const float nm = fmaxf(M, c[u].x);
          S = S * es_exp(M - nm) + c[u].y * es_exp(c[u].x - nm);   // exp(-inf) = 0 on the first chunk
          M = nm;
        }
      }
    }
    for (int st = 16; st >= H; st >>= 1) {
      const float oM = __shfl_xor_sync(FULL, M, st), oS = __shfl_xor_sync(FULL, S, st);
      if (MODE == 1 || MODE == 3) {
        S += oS;
      } else {
        const float nm = fmaxf(M, oM);
        const float a = (M == -CUDART_INF_F) ? 0.f : S * es_exp(M - nm);
        const float b = (oM == -CUDART_INF_F) ? 0.f : oS * es_exp(oM - nm);
        S = a + b;
        M = nm;
      }
    }
    __syncwarp();
    if (lane < H) {
      float2 *dst = p.stats + (int64_t)w.first * H + lane;
      asm volatile("st.global.cg.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(M), "f"(S) : "memory");
    }
  }
}

// ---------------------------------------------------------------- hub chunk, pass 2 (a chunk item of the main kernel)
// normalise the chunk's elements with its row's merged statistics (stats[first slot])
template <int MODE, bool DROP, bool TYPED, bool MIX>
__device__ __forceinline__ void es_chunk_item(const EsParams &p, const float *tab, int64_t item, int lane) {
  constexpr bool TWO = (MODE == 1 || MODE == 3);
  const int H = p.H;

    const WorkItem w = decode_item(item, 0, p.rowptr, p.hub);
    const int head = lane & (H - 1);
    const int n = (w.hb - w.lb) * H;
    const float2 rs = __ldcg(p.stats + (int64_t)w.first * H + head);
    float *o = p.out + (int64_t)w.lb * H;
    if (TWO) {
      const float *y = p.a + (int64_t)w.lb * H, *g = p.b + (int64_t)w.lb * H;
      if (MODE == 1) {
#pragma unroll 4
        for (int t = lane; t < n; t += 32) st_stream(o + t, __ldg(y + t) * (__ldg(g + t) - rs.y));
      } else {
        const float hlrow = __ldg(p.hl + (int64_t)w.row * H + head);
        float acc = 0.f;
        for (int t = lane; t < n; t += 32) {
          float yv = __ldg(y + t), gv = __ldg(g + t);
          es_unmark<DROP>(p, yv, gv);
          const float v = yv * (gv - rs.y) * es_dact<TYPED>(p, tab, w.lb, t, head, hlrow);
          st_stream(o + t, v);
          acc += v;
        }
        acc = head_sum(acc, H);
        if (lane < H) st_cg(p.part + (int64_t)w.slot * H + lane, acc);
        if (hub_arrive_last<32>(w, p.hub, lane)) {      // row sum of the hub row: chunk partials in chunk order
          if (lane < H) {
            float tot = 0.f;
            for (int q = 0; q < w.n_row_chunks; ++q) tot += ld_cg(p.part + (int64_t)(w.first + q) * H + lane);
            p.grow[(int64_t)w.row * H + lane] = tot;
          }
        }
      }
    } else {
      const float hl = (MODE == 2) ? __ldg(p.a + (int64_t)w.row * H + head) : 0.f;
      const float inv = 1.f / rs.y;
      const int64_t ob = (int64_t)w.lb * H;
#pragma unroll 4
      for (int t = lane; t < n; t += 32)
        es_put<TYPED, MIX>(p, ob + t, es_mark<DROP>(p, w.lb + (t >> p.lgH), head,
                                                    es_exp(es_in<MODE, TYPED>(p, tab, w.lb, t, head, hl) - rs.x) * inv));
    }
    }

// ---------------------------------------------------------------- bulk-copy helpers (TMA 1-D)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared, completion counted in bytes on the mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// shared -> global, tracked by the bulk async-group of the issuing thread
__device__ __forceinline__ void bulk_s2g(void *dst, const void *src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- main kernel: chunks + segments
// Warps per block of the main kernel.  For the 512-float tile this is a launch parameter only (2 and 4 warps give
// bit-identical outputs); a block's shared memory and warp slots are released when its slowest warp retires, and 8
// is the shape the whole GPU suite is validated with.
constexpr int ES_WARPS = 8;

// Dynamic shared memory per warp: CAP floats (+ CAP for the backward's second operand) + 33 row offsets.
template <int MODE, int CAP, bool DROP, bool TYPED, bool MIX>
__global__ void __launch_bounds__(ES_WARPS * 32) es_main_kernel(const EsParams p) {
  __shared__ float table[TYPED ? HGN_MAX_TABLE : 1];
  const float *tab = es_stage_table<TYPED>(p, table);
  constexpr bool TWO = (MODE == 1 || MODE == 3);
  extern __shared__ __align__(128) unsigned char es_smem[];
  float *tiles = reinterpret_cast<float *>(es_smem);
  int *rps = reinterpret_cast<int *>(es_smem + (size_t)ES_WARPS * CAP * 4 * (TWO ? 2 : 1));
  uint64_t *bars = reinterpret_cast<uint64_t *>(rps + ES_WARPS * 34);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t item = (int64_t)blockIdx.x * ES_WARPS + wib;
  const int H = p.H;

  // ------------------------------------------------ hub chunk (LAST in the grid): normalise with the row's merged
  // statistics, which the statistics kernel -- possibly still running: programmatic dependent launch -- produces
  if (item >= p.hub.n_segs) {
    if (item - p.hub.n_segs < p.hub.n_chunks) {
      asm volatile("griddepcontrol.wait;" ::: "memory");
      es_chunk_item<MODE, DROP, TYPED, MIX>(p, tab, item - p.hub.n_segs, lane);
    }
    return;
  }

  // ------------------------------------------------ segment of short rows
  const int64_t seg = item;
  const int2 rr = __ldg(p.hub.segs + seg);
  float *T = tiles + (size_t)wib * CAP * (TWO ? 2 : 1);
  float *T2 = T + CAP;
  int *RP = rps + wib * 34;
  uint64_t *bar = bars + wib;
  const bool bulk = p.bulk && MODE != 2;
  if (bulk) {
    if (lane == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
  }
  uint32_t phase = 0;
  int rw = rr.x;
  while (rw < rr.y) {
    // window of <= 32 rows starting at rw; keep the longest prefix that fits the tile
    const int row = rw + lane;
    const int base = __ldg(p.rowptr + rw);
    int endl = 0x7fffffff;
    if (row < rr.y) endl = __ldg(p.rowptr + row + 1);
    const unsigned fit = __ballot_sync(FULL, row < rr.y && (int64_t)(endl - base) * H <= CAP);
    const int m = __popc(fit);                 // fit is a prefix mask (row ends are monotone)
    if (m == 0) {                              // cannot happen when chunk_edges * H <= CAP (host check)
      rw += 1;
      continue;
    }
    const int e_end = __shfl_sync(FULL, endl, m - 1);
    const int n = (e_end - base) * H;
    // ---- stage (issue the bulk copy first, do the index work while it flies)
    if (bulk && n > 0) {
      if (lane == 0) {
        mbar_expect_tx(bar, (uint32_t)n * 4u * (TWO ? 2u : 1u));
        bulk_g2s(T, p.a + (int64_t)base * H, (uint32_t)n * 4u, bar);
        if (TWO) bulk_g2s(T2, p.b + (int64_t)base * H, (uint32_t)n * 4u, bar);
      }
    }
    const int startl = __shfl_up_sync(FULL, endl, 1);
    const int sl = (lane == 0) ? base : startl;          // start edge of my row
    if (lane < m) RP[lane + 1] = endl - base;
    if (lane == 0) RP[0] = 0;
    // degree-sorted visiting order of the window's rows (ascending): key = degree << 5 | row slot
    unsigned key = (lane < m) ? (((unsigned)(endl - sl) << 5) | (unsigned)lane) : 0xffffffffu;
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
      for (int j = k >> 1; j > 0; j >>= 1) {
        const unsigned o = __shfl_xor_sync(FULL, key, j);
        const bool up = (lane & k) == 0, lower = (lane & j) == 0;
        key = (lower == up) ? min(key, o) : max(key, o);
      }
    }
    if (!bulk) {
      if (MODE == 2) {
#pragma unroll 4
        for (int t = lane; t < n; t += 32) {
          const int pe = base + (t >> p.lgH), h = t & (H - 1);
          const int r = __ldg(p.hub.edge_row + pe);
          const int c = __ldg(p.colind + pe);
          const float z = es_typed<TYPED>(p, tab, pe, h, __ldg(p.a + (int64_t)r * H + h) + __ldg(p.b + (int64_t)c * H + h));
          T[t] = z > 0.f ? z : z * p.slope;
        }
      } else {
        const float *src = p.a + (int64_t)base * H;
#pragma unroll 4
        for (int t = lane; t < n; t += 32) T[t] = ld_stream(src + t);
        if (TWO) {
          const float *src2 = p.b + (int64_t)base * H;
#pragma unroll 4
          for (int t = lane; t < n; t += 32) T2[t] = ld_stream(src2 + t);
        }
      }
    }
    __syncwarp();
    if (bulk && n > 0) {
      mbar_wait(bar, phase);
      phase ^= 1u;
    }
    // ---- (row, head) pairs, rows in degree-sorted order (warp-uniform trip count: the shuffle needs all lanes)
    const int pairs = m * H;
    for (int q0 = 0; q0 < pairs; q0 += 32) {
      const int q = q0 + lane;
      const int rl = (int)(__shfl_sync(FULL, key, min(q >> p.lgH, 31)) & 31u);
      if (q < pairs) {
        const int h = q & (H - 1);
        const int k0 = RP[rl], k1 = RP[rl + 1];
        if (TWO) {
          float s = 0.f;
          for (int k = k0; k < k1; ++k) {
            float yv = T[k * H + h], gv = T2[k * H + h];
            es_unmark<DROP>(p, yv, gv);
            s = fmaf(yv, gv, s);
          }
          if (MODE == 1) {
            for (int k = k0; k < k1; ++k) T[k * H + h] = T[k * H + h] * (T2[k * H + h] - s);
          } else {
            const int grow_row = rw + rl;
            const float hlrow = __ldg(p.hl + (int64_t)grow_row * H + h);
            float acc = 0.f;
            for (int k = k0; k < k1; ++k) {
              const int c = __ldg(p.colind + base + k);
              const float z = es_typed<TYPED>(p, tab, base + k, h, hlrow + __ldg(p.hr + (int64_t)c * H + h));
              float yv = T[k * H + h], gv = T2[k * H + h];
              es_unmark<DROP>(p, yv, gv);
              const float v = yv * (gv - s) * (z > 0.f ? 1.f : p.slope);
              T[k * H + h] = v;
              acc += v;
            }
            p.grow[(int64_t)grow_row * H + h] = acc;     // also the (empty-row) zero
          }
        } else {
          // online max / sum (one pass, one exp per element: e = exp(-|x - m|) is the rescale factor of the running
          // sum when x is a new maximum and the new term otherwise), then one normalising pass: 2 LDS + 1 STS and
          // 2 MUFU per element instead of 3 LDS + 2 STS -- the kernel is issue-bound.  The running max starts at
          // -FLT_MAX, not -inf: a leading -inf logit then gives d = -inf and e = 0 instead of -inf - -inf = NaN, and
          // a (row, head) whose logits are all -inf still ends in 0 * (1 / 0) = NaN, as the softmax does.
          float mx = -FLT_MAX, sm = 0.f;
          for (int k = k0; k < k1; ++k) {
            const float x = T[k * H + h];
            const float d = x - mx;
            const float e = es_exp(-fabsf(d));
            sm = (d > 0.f) ? fmaf(sm, e, 1.f) : sm + e;
            mx = fmaxf(mx, x);
          }
          // a +Inf logit became the max and counted as exp(0) = 1, but the softmax has exp(Inf - Inf) = NaN there:
          // the whole (row, head) is NaN, as it is on the unsegmented and chunked paths
          const float inv = mx < CUDART_INF_F ? 1.f / sm : CUDART_NAN_F;
          for (int k = k0; k < k1; ++k) T[k * H + h] = es_mark<DROP>(p, (int64_t)base + k, h, es_exp(T[k * H + h] - mx) * inv);
        }
      }
    }
    __syncwarp();
    // ---- write back
    float *dst = p.out + (int64_t)base * H;
    if (bulk && n > 0) {
      fence_async_smem();                      // my generic-proxy writes to T -> visible to the async proxy
      __syncwarp();
      if (lane == 0) {
        bulk_s2g(dst, T, (uint32_t)n * 4u);
        bulk_commit();
        bulk_wait_read0();                     // T may be overwritten (next window) / freed (exit) after this
      }
      __syncwarp();
    } else if (MODE == 2) {
      for (int t = lane; t < n; t += 32) es_put<TYPED, MIX>(p, (int64_t)base * H + t, T[t]);
      __syncwarp();
    } else {
      for (int t = lane; t < n; t += 32) st_stream(dst + t, T[t]);
      __syncwarp();
    }
    rw += m;
  }
}

// ---------------------------------------------------------------- generic H: warp per row, loop over heads
template <int MODE, bool DROP, bool TYPED, bool MIX>
__global__ void __launch_bounds__(256) es_generic_kernel(const EsParams p) {
  __shared__ float table[TYPED ? HGN_MAX_TABLE : 1];
  const float *tab = es_stage_table<TYPED>(p, table);
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= p.n_rows) return;
  const int lb = __ldg(p.rowptr + row), hb = __ldg(p.rowptr + row + 1);
  for (int h = 0; h < p.H; ++h) {
    if (MODE == 1 || MODE == 3) {
      float s = 0.f;
      for (int e = lb + lane; e < hb; e += 32) {
        float yv = __ldg(p.a + (int64_t)e * p.H + h), gv = __ldg(p.b + (int64_t)e * p.H + h);
        es_unmark<DROP>(p, yv, gv);
        s = fmaf(yv, gv, s);
      }
      s = head_sum(s, 1);
      const float hlrow = (MODE == 3) ? __ldg(p.hl + row * p.H + h) : 0.f;
      float acc = 0.f;
      for (int e = lb + lane; e < hb; e += 32) {
        const int64_t k = (int64_t)e * p.H + h;
        float yv = __ldg(p.a + k), gv = __ldg(p.b + k);
        es_unmark<DROP>(p, yv, gv);
        float v = yv * (gv - s);
        if (MODE == 3) {
          const float z = es_typed<TYPED>(p, tab, e, h, hlrow + __ldg(p.hr + (int64_t)__ldg(p.colind + e) * p.H + h));
          v *= (z > 0.f ? 1.f : p.slope);
          acc += v;
        }
        p.out[k] = v;
      }
      if (MODE == 3) {
        acc = head_sum(acc, 1);
        if (lane == 0) p.grow[row * p.H + h] = acc;
      }
    } else {
      const float hl = (MODE == 2) ? __ldg(p.a + row * p.H + h) : 0.f;
      auto in = [&](int e) {
        if (MODE == 2) {
          const float z = es_typed<TYPED>(p, tab, e, h, hl + __ldg(p.b + (int64_t)__ldg(p.colind + e) * p.H + h));
          return z > 0.f ? z : z * p.slope;
        }
        return __ldg(p.a + (int64_t)e * p.H + h);
      };
      float m = -CUDART_INF_F;
      for (int e = lb + lane; e < hb; e += 32) m = fmaxf(m, in(e));
      m = head_max(m, 1);
      float s = 0.f;
      for (int e = lb + lane; e < hb; e += 32) s += expf(in(e) - m);
      s = head_sum(s, 1);
      for (int e = lb + lane; e < hb; e += 32) {
        const float a = es_mark<DROP>(p, e, h, expf(in(e) - m) / s);
        if (TYPED) es_put<TYPED, MIX>(p, (int64_t)e * p.H + h, a);
        else p.out[(int64_t)e * p.H + h] = a;
      }
    }
  }
}

// Launch the main kernel (segments first, hub chunks last) on the items of p's plan.
template <int MODE, int CAP, bool DROP, bool TYPED, bool MIX>
static int es_launch_main(const EsParams &p, cudaStream_t s) {
  const auto kernel = es_main_kernel<MODE, CAP, DROP, TYPED, MIX>;
  // per warp: the tile(s), the row offsets and the mbarrier
  constexpr size_t smem = (size_t)ES_WARPS * CAP * 4 * ((MODE == 1 || MODE == 3) ? 2 : 1) + (size_t)ES_WARPS * 34 * 4 +
                          (size_t)ES_WARPS * 8;
  static unsigned long long attr_done = 0;   // the kernel's per-device record of its shared-memory attribute
  int dev = 0;
  if (first_use_on_device(attr_done, &dev))
    CB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t items = (int64_t)p.hub.n_chunks + p.hub.n_segs;
  const int64_t blocks = ceil_div(items, ES_WARPS);
  if (blocks == 0) return COGDL_B200_OK;
  CB_REQUIRE(blocks <= 0x7fffffffLL, "edge_softmax: problem too large for one launch");
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3(ES_WARPS * 32);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;   // overlap with the statistics kernel (see es_stats_kernel)
  cfg.attrs = attr;
  cfg.numAttrs = p.hub.n_chunks > 0 ? 1 : 0;
  CB_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
  count_launch();
  return COGDL_B200_OK;
}

// The launch form a call takes (see the header comment of edge_softmax.cu).
enum class EsForm { GENERIC, WARP, MAIN };

// Fill the plan-dependent fields of p (lgH, hub, stats, part, bulk) and choose the launch form; for MAIN, *cap is the
// smallest tile (floats per warp) that fits a chunk.  Returns nonzero (and sets the error) when the plan's scratch is
// too small.
template <int MODE>
static int es_plan(EsParams &p, const cogdl_b200_hub_plan_t *plan, EsForm *form, int *cap) {
  const bool pow2 = p.H <= 32 && (p.H & (p.H - 1)) == 0;
  p.lgH = 0;
  while ((1 << p.lgH) < p.H) ++p.lgH;
  p.hub = hub_view(nullptr);
  p.stats = nullptr; p.part = nullptr; p.bulk = false;
  *cap = 0;
  if (!pow2) {
    *form = EsForm::GENERIC;
    return COGDL_B200_OK;
  }
  const int64_t cap_need = plan ? (int64_t)plan->chunk_edges * p.H : 0;
  const bool segs = plan && plan->chunk_edges > 0 && plan->segs && plan->edge_row && plan->n_segs > 0 && cap_need <= 2048;
  if (!segs) {   // no plan: every row through the warp kernel (hubs serialise on one warp)
    *form = EsForm::WARP;
    return COGDL_B200_OK;
  }
  p.hub = hub_view(plan);
  // scratch: (max, sum) per chunk slot and head, then (MODE 3) one partial row sum per slot and head
  int rc = check_plan(plan, cogdl_b200_edge_softmax_scratch_bytes(p.hub.n_chunks, p.H));
  if (rc) return rc;
  p.stats = reinterpret_cast<float2 *>(plan->partials);
  p.part = reinterpret_cast<float *>(p.stats + (int64_t)p.hub.n_chunks * p.H);
  // 1-D TMA needs 16-byte aligned global addresses and sizes: rows start at multiples of H floats
  p.bulk = (p.H % 4 == 0) && aligned16(p.a) && aligned16(p.out) && (MODE == 0 || aligned16(p.b));
  *form = EsForm::MAIN;
  *cap = cap_need <= 512 ? 512 : (cap_need <= 1024 ? 1024 : 2048);
  return COGDL_B200_OK;
}

// The launch plan (see the header comment of edge_softmax.cu).  The typed MODE 3 always reads the signed attention
// (DROP): its gradient scale applies with or without dropout.  cogdl_b200_last_kernel() records the launches as
// es_*_kernel, or hgn_*_kernel when TYPED; of the two name formats only the es_ one names the main kernel's warps per
// block, and the DROP of the MODE-3 statistics kernel.
template <int MODE, bool DROP, bool TYPED, bool MIX>
static int es_launch(EsParams p, const cogdl_b200_hub_plan_t *plan, cudaStream_t s, const char *who) {
  static_assert(!DROP || MODE == 2 || MODE == 3, "attention dropout is a mode of the GAT attention and its backward");
  static_assert(TYPED ? MODE == 2 || (MODE == 3 && DROP && !MIX) : !MIX,
                "the typed kernels are the attention and its backward, and only the typed attention blends");
  const char *fam = TYPED ? "hgn" : "es";
  const char *flags = DROP ? (MIX ? ",DROP,MIX" : ",DROP") : (MIX ? ",MIX" : "");
  const int64_t row_blocks = ceil_div(p.n_rows * 32, 256);
  CB_REQUIRE(row_blocks <= 0x7fffffffLL, "%s: problem too large for one launch", who);
  EsForm form;
  int chosen;
  int rc = es_plan<MODE>(p, plan, &form, &chosen);
  if (rc) return rc;
  if (form == EsForm::GENERIC) {
    note_kernel("cogdl_b200::%s_generic_kernel<MODE=%d%s>", fam, MODE, flags);
    es_generic_kernel<MODE, DROP, TYPED, MIX><<<(unsigned)row_blocks, 256, 0, s>>>(p);
    CB_LAUNCH_CHECK();
    return COGDL_B200_OK;
  }
  if (form == EsForm::WARP) {
    note_kernel("cogdl_b200::%s_warp_kernel<MODE=%d%s>", fam, MODE, flags);
    es_warp_kernel<MODE, DROP, TYPED, MIX><<<(unsigned)row_blocks, 256, 0, s>>>(p);
    CB_LAUNCH_CHECK();
    return COGDL_B200_OK;
  }
  // both launches, in launch order, when the statistics kernel runs
  char stats_note[64] = "";
  if (p.hub.n_chunks > 0) {
    // the attention's statistics come before the dropout: MODE 2 shares the kernel without DROP
    constexpr bool SDROP = DROP && MODE == 3;
    es_stats_kernel<MODE, SDROP, TYPED><<<(unsigned)ceil_div((int64_t)p.hub.n_chunks * 32, 256), 256, 0, s>>>(p);
    CB_LAUNCH_CHECK();
    snprintf(stats_note, sizeof(stats_note), "cogdl_b200::%s_stats_kernel<MODE=%d%s> + ", fam, MODE,
             (SDROP && !TYPED) ? ",DROP" : "");
  }
  char warps[16] = "";
  if (!TYPED) snprintf(warps, sizeof(warps), ",WARPS=%d", ES_WARPS);
  note_kernel("%scogdl_b200::%s_main_kernel<MODE=%d,CAP=%d%s%s>%s", stats_note, fam, MODE, chosen, warps, flags,
              (p.bulk && MODE != 2) ? " cp.async.bulk tiles" : "");
  if (chosen == 512) return es_launch_main<MODE, 512, DROP, TYPED, MIX>(p, s);
  if (chosen == 1024) return es_launch_main<MODE, 1024, DROP, TYPED, MIX>(p, s);
  return es_launch_main<MODE, 2048, DROP, TYPED, MIX>(p, s);
}

}  // namespace cogdl_b200

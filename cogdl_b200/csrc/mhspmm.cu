// mhspmm.cu -- multi-head SpMM (GAT aggregation) for sm_90a.
//
//   out[i,h,:] = sum_{p in row i} att[P(p),h] * feat[colind[p],h,:]      P(p) = perm ? perm[p] : p
//
// Replaces mhspmmSimple / mhspmm_1 (cogdl/operators/spmm/multiheadSpmm.cu:6-51): grid (V,H) with
// F-thread blocks => rowptr/colind re-read H times, one dependent colind->feat load chain per
// edge, F=16 gives half-warp blocks.  `perm` additionally fuses the backward's mhtranspose
// (mhTranspose.cu:6-49, mhspmm.py:60-61) so the CSC pass never materialises att[perm].
//
// A node's [H,F] block is one contiguous run of H*F floats.  It is cut into slices of GROUP
// 16-byte vectors (512 B for GROUP = 32); a GROUP of lanes owns one (row-or-hub-chunk, slice)
// item, slices of the same row sit in adjacent warps so the index/attention lines they share
// are L1 hits.  The lane's head is fixed (its column / F), its attention scalar is fetched per
// edge next to the feature gather (same 32-byte sector for all lanes of a head).  Accumulation
// order and rounding are those of the SpMM (CSR order, separate fp32 mul and add), i.e. the
// reference's CPU fallback (one spmm_cpu per head, spmm_utils.py:216-225).
#include "common.cuh"
#include "stream.cuh"

#include <cstdio>

namespace cogdl_b200 {

struct MhParams {
  const int *rowptr;
  const int *colind;
  const int *perm;   // nullable
  const float *att;  // [nnz, H]
  const float *feat; // [n_src, H*F]
  float *out;        // [n_rows, H*F]
  int64_t n_rows;
  int H;
  int HFV;           // H*F in vector units
  int FVL;           // F in vector units  (head = col / FVL)
  int S;             // slices per row
  HubView hub;
  float drop_scale;  // > 0: att carries an attention-dropout mask in its sign bit (drop_att); 0: plain attention
};

template <typename VecT, int GROUP, bool HAS_PERM, bool DROP>
__global__ void __launch_bounds__(256) mhspmm_kernel(const MhParams p) {
  constexpr int U0 = 8;
  constexpr int U = U0 < GROUP ? U0 : GROUP;
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t gidx = tid / GROUP;
  const int64_t item = gidx / p.S;
  const int slice = (int)(gidx - item * p.S);
  const WorkItem w = decode_item(item, p.n_rows, p.rowptr, p.hub);
  const bool warp_has_chunk = ((tid - lane) / GROUP) / p.S < p.hub.n_chunks;

  const int cv = slice * GROUP + gl;
  const bool colok = cv < p.HFV;
  const int head = colok ? cv / p.FVL : 0;
  const VecT *X = reinterpret_cast<const VecT *>(p.feat);
  VecT *Y = reinterpret_cast<VecT *>(p.out);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);

  VecT acc = vzero<VecT>();
  int c = 0, pe = 0;
  {
    const int e = w.lb + gl;
    if (e < w.hb) {
      c = ld_stream(p.colind + e);
      pe = HAS_PERM ? ld_stream(p.perm + e) : e;
    }
  }
  for (int off = 0; off < maxdeg; off += GROUP) {
    const int cnt = min(GROUP, w.hb - w.lb - off);
    int cn = 0, pn = 0;
    {
      const int e = w.lb + off + GROUP + gl;
      if (e < w.hb) {
        cn = ld_stream(p.colind + e);
        pn = HAS_PERM ? ld_stream(p.perm + e) : e;
      }
    }
#pragma unroll 1
    for (int j = 0; j < GROUP; j += U) {
      if (GROUP == 32) {
        if (j >= cnt) break;
      } else {
        if (!__any_sync(FULL, j < cnt)) break;
      }
      VecT x[U];
      float a[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int cj = __shfl_sync(FULL, c, j + u, GROUP);
        const int pj = __shfl_sync(FULL, pe, j + u, GROUP);
        if (j + u < cnt && colok) {
          x[u] = ld_gather(X + (int64_t)cj * p.HFV + cv);
          a[u] = __ldg(p.att + (int64_t)pj * p.H + head);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (j + u < cnt && colok) axpy_rn(acc, DROP ? drop_att(a[u], p.drop_scale) : a[u], x[u]);
    }
    c = cn;
    pe = pn;
  }

  if (!w.is_chunk) {
    if (w.active && colok) st_stream(Y + (int64_t)w.row * p.HFV + cv, acc);
  } else if (colok) {
    st_cg(P + (int64_t)w.slot * p.HFV + cv, acc);
  }
  if (warp_has_chunk) {
    // all S slice-groups of every chunk of the row arrive on one counter; the last one of all
    // combines the whole row (every slice) in chunk order
    WorkItem wa = w;
    wa.n_row_chunks = w.n_row_chunks * p.S;
    if (hub_arrive_last<GROUP>(wa, p.hub, gl)) {
      for (int k = gl; k < p.HFV; k += GROUP) {
        const VecT *pp = P + (int64_t)w.first * p.HFV + k;
        const VecT s = merge_chunks<1>(w.n_row_chunks, [&](int q) { return ld_cg(pp + (int64_t)q * p.HFV); },
                                       [](VecT &a, const VecT &t) { add_rn(a, t); });
        st_stream(Y + (int64_t)w.row * p.HFV + k, s);
      }
    }
  }
}

template <typename VecT, int GROUP>
static int launch_mh(const MhParams &p, cudaStream_t stream) {
  const bool drop = p.drop_scale > 0.f;
  auto kernel = drop ? (p.perm ? mhspmm_kernel<VecT, GROUP, true, true> : mhspmm_kernel<VecT, GROUP, false, true>)
                     : (p.perm ? mhspmm_kernel<VecT, GROUP, true, false> : mhspmm_kernel<VecT, GROUP, false, false>);
  return launch_items(kernel, p, ((int64_t)p.hub.n_chunks + p.n_rows) * p.S, GROUP, stream, "mhspmm",
                      "cogdl_b200::mhspmm_kernel<%s,GROUP=%d,%s%s>", sizeof(VecT) == 16 ? "float4" : "float", GROUP,
                      p.perm ? "perm" : "no_perm", drop ? ",drop" : "");
}

template <typename VecT>
static int dispatch_mh(MhParams &p, cudaStream_t s) {
  const int n = p.HFV;
  int g = 1;
  while (g < 32 && g < n) g <<= 1;
  p.S = (int)ceil_div(n, g);
  if (g == 32 && p.hub.n_segs > 0) {
    // row-stream form: one warp per (segment or hub chunk, 512-byte slice)
    StreamParams q;
    q.rowptr = p.rowptr; q.colind = p.colind; q.val = nullptr; q.att = p.att; q.perm = p.perm;
    q.X0 = p.feat; q.X1 = p.feat; q.n0 = INT64_MAX; q.Y = p.out; q.ldv = p.HFV; q.H = p.H; q.FVL = p.FVL;
    q.S = p.S; q.hub = p.hub; q.n_peers = 0; q.peer_shift = 0; q.drop_scale = p.drop_scale;
    return launch_stream<VecT, 1, 8, 3, true, FORM_MULTIHEAD>(q, s);
  }
  switch (g) {
    case 1: return launch_mh<VecT, 1>(p, s);
    case 2: return launch_mh<VecT, 2>(p, s);
    case 4: return launch_mh<VecT, 4>(p, s);
    case 8: return launch_mh<VecT, 8>(p, s);
    case 16: return launch_mh<VecT, 16>(p, s);
    default: return launch_mh<VecT, 32>(p, s);
  }
}

// drop_scale > 0: att carries an attention-dropout mask in its sign bit (see drop_att); 0: plain attention.
static int mhspmm_run(const int32_t *rowptr, const int32_t *colind, const int32_t *perm, const float *att,
                      const float *feat, float *out, int64_t n_rows, int64_t H, int64_t F,
                      const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream, float drop_scale = 0.f) {
  MhParams p;
  p.rowptr = rowptr; p.colind = colind; p.perm = perm; p.att = att; p.feat = feat; p.out = out;
  p.n_rows = n_rows; p.H = (int)H; p.hub = hub_view(plan); p.S = 1; p.drop_scale = drop_scale;
  const bool vec = (F % 4 == 0) && aligned16(feat) && aligned16(out) &&
                   (p.hub.n_chunks == 0 || aligned16(p.hub.partials));
  if (vec) {
    p.HFV = (int)(H * F / 4);
    p.FVL = (int)(F / 4);
    return dispatch_mh<float4>(p, (cudaStream_t)stream);
  }
  p.HFV = (int)(H * F);
  p.FVL = (int)F;
  return dispatch_mh<float>(p, (cudaStream_t)stream);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_mhspmm_scratch_bytes(int64_t n_chunks, int64_t H, int64_t F) {
  return n_chunks > 0 && H > 0 && F > 0 ? n_chunks * H * F * (int64_t)sizeof(float) : 0;
}

static int mhspmm_entry(const int32_t *rowptr, const int32_t *colind, const int32_t *perm, const float *att,
                        const float *feat, float *out, int64_t n_rows, int64_t H, int64_t F,
                        const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream, float drop_scale,
                        const char *who) {
  CB_REQUIRE(n_rows >= 0 && H >= 0 && F >= 0, "%s: negative size", who);
  if (n_rows == 0 || H == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && att && feat && out, "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && H * F < 0x7fffffffLL, "%s: sizes must fit int32", who);
  int rc = check_plan(plan, cogdl_b200_mhspmm_scratch_bytes(plan ? plan->n_chunks : 0, H, F));
  if (rc) return rc;
  return mhspmm_run(rowptr, colind, perm, att, feat, out, n_rows, H, F, plan, stream, drop_scale);
}

extern "C" int cogdl_b200_mhspmm_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                                     const float *att, const float *feat, float *out, int64_t n_rows,
                                     int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                     cogdl_b200_stream_t stream) {
  return mhspmm_entry(rowptr, colind, perm, att, feat, out, n_rows, H, F, plan, stream, 0.f, "cogdl_b200_mhspmm_f32");
}

// The aggregation over an attention written by cogdl_b200_gat_fwd_dropout_f32: entries with the sign bit set are
// dropped, the others are scaled by `scale`.  With perm (the cached transpose) this is d feat of the dropout GAT.
extern "C" int cogdl_b200_mhspmm_dropout_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                                             const float *att, const float *feat, float scale, float *out,
                                             int64_t n_rows, int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                             cogdl_b200_stream_t stream) {
  CB_REQUIRE(isfinite(scale) && scale > 0.f, "cogdl_b200_mhspmm_dropout_f32: scale must be finite and > 0 (got %g)",
             (double)scale);
  return mhspmm_entry(rowptr, colind, perm, att, feat, out, n_rows, H, F, plan, stream, scale,
                      "cogdl_b200_mhspmm_dropout_f32");
}

// ------------------------------------------------------------------------------------------
// GAT forward (SURVEY 8f-1):   e[p,h] = leakyrelu(h_l[i,h] + h_r[colind[p],h])   (p in row i)
//                              a[p,:] = softmax over the row's edges, per head
//                              out[i,h] = sum_p a[p,h] * feat[colind[p],h,:]
// Replaces the unfused chain of cogdl/layers/gat_layer.py:73-77 (two [nnz,H] gathers, an add, a LeakyReLU and a
// softmax, each a kernel with its own [nnz,H] temporary) and the stale dgNN binding (cogdl/operators/fused_gat.py:
// 17-19; precedent third_party/dgNN/.../fused_gatconv_kernel.cu:26-133).  Two stages on the caller's stream:
//   1. attention (edge_softmax.cu, MODE 2): logits formed from h_l / h_r while loading and soft-maxed per row in
//      the same pass; only the normalised attention [nnz,H] is written -- it is also what the backward saves;
//   2. the row-stream multi-head SpMM above consumes it (0.97 of the HBM roofline at H=8, F=128, so a single-pass
//      fusion could only remove the 8*H-byte attention round trip per edge against 4*H*F bytes of gather: 1.6 %;
//      round 1's per-(row, slice) fully fused kernel recomputed the statistics per slice and was 4x slower).
// The backward is native as well: see cogdl_b200_gat_attn_bwd_f32 (edge_softmax.cu) and operators/fused_gat.py.
// ------------------------------------------------------------------------------------------
namespace cogdl_b200 {
int gat_attention(const int32_t *rowptr, const int32_t *colind, const float *h_l, const float *h_r, float slope,
                  float *att, int64_t n_rows, int64_t H, const cogdl_b200_hub_plan_t *plan, cudaStream_t s,
                  bool drop, uint64_t seed, uint64_t drop_below);
}

// The attention stage and the aggregation use the same partials one after the other.
extern "C" int64_t cogdl_b200_gat_fwd_scratch_bytes(int64_t n_chunks, int64_t H, int64_t F) {
  const int64_t att = cogdl_b200_edge_softmax_scratch_bytes(n_chunks, H);
  const int64_t agg = cogdl_b200_mhspmm_scratch_bytes(n_chunks, H, F);
  return att > agg ? att : agg;
}

// drop: attention dropout (seed, drop_below, scale) -- see cogdl_b200_gat_fwd_dropout_f32
static int gat_fwd(const int32_t *rowptr, const int32_t *colind, const float *h_l, const float *h_r, const float *feat,
                   float negative_slope, bool drop, uint64_t seed, uint64_t drop_below, float scale, float *out,
                   float *att_out, int64_t n_rows, int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan,
                   cogdl_b200_stream_t stream, const char *who) {
  CB_REQUIRE(n_rows >= 0 && H >= 0 && F >= 0, "%s: negative size", who);
  if (n_rows == 0 || H == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && h_l && h_r && feat && out, "%s: null pointer", who);
  CB_REQUIRE(att_out, "%s: att_out ([nnz,H] attention, also scratch) is required", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && H * F < 0x7fffffffLL, "%s: sizes must fit int32", who);
  int rc = check_plan(plan, cogdl_b200_gat_fwd_scratch_bytes(plan ? plan->n_chunks : 0, H, F));
  if (rc) return rc;
  rc = gat_attention(rowptr, colind, h_l, h_r, negative_slope, att_out, n_rows, H, plan, (cudaStream_t)stream, drop,
                     seed, drop_below);
  if (rc) return rc;
  // cogdl_b200_last_kernel() names both stages: "<attention> + <aggregation>" (each note is under 128 bytes)
  char att_note[128], agg_note[128];
  snprintf(att_note, sizeof(att_note), "%s", cogdl_b200_last_kernel());
  rc = mhspmm_run(rowptr, colind, nullptr, att_out, feat, out, n_rows, H, F, plan, stream, drop ? scale : 0.f);
  if (rc) return rc;
  snprintf(agg_note, sizeof(agg_note), "%s", cogdl_b200_last_kernel());
  note_kernel("%s + %s", att_note, agg_note);
  return COGDL_B200_OK;
}

extern "C" int cogdl_b200_gat_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *h_l,
                                      const float *h_r, const float *feat, float negative_slope, float *out,
                                      float *att_out, int64_t n_rows, int64_t H, int64_t F,
                                      const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return gat_fwd(rowptr, colind, h_l, h_r, feat, negative_slope, false, 0, 0, 0.f, out, att_out, n_rows, H, F, plan,
                 stream, "cogdl_b200_gat_fwd_f32");
}

// GAT forward with attention dropout: (edge p, head h) is kept iff draw(seed, p, h) >= drop_below (rng.cuh), and a
// kept attention is scaled by `scale` in the aggregation.  att_out holds the softmax with the sign bit set on the
// dropped entries -- the mask travels to the backward in the saved attention, nothing else is stored.
extern "C" int cogdl_b200_gat_fwd_dropout_f32(const int32_t *rowptr, const int32_t *colind, const float *h_l,
                                              const float *h_r, const float *feat, float negative_slope, uint64_t seed,
                                              uint64_t drop_below, float scale, float *out, float *att_out,
                                              int64_t n_rows, int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                              cogdl_b200_stream_t stream) {
  CB_REQUIRE(isfinite(scale) && scale > 0.f, "cogdl_b200_gat_fwd_dropout_f32: scale must be finite and > 0 (got %g)",
             (double)scale);
  return gat_fwd(rowptr, colind, h_l, h_r, feat, negative_slope, true, seed, drop_below, scale, out, att_out, n_rows,
                 H, F, plan, stream, "cogdl_b200_gat_fwd_dropout_f32");
}

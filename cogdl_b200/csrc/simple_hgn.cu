// simple_hgn.cu -- Simple-HGN attention (myGATConv of CogDL's examples/simple_hgn/conv.py) for sm_90a: the GAT
// attention stage of edge_softmax.cu with an edge-type term in the logit and the residual attention blend in the
// store, and its backward.
//
// Forward, per CSR edge p = (i, j) of type t = type[p] and head h:
//   a[p,h]   = softmax over row i of leakyrelu(h_l[i,h] + h_r[j,h] + h_e[t,h])
//   att[p,h] = a, with the sign bit set when dropped (the GAT-dropout carrier: the same mask, seed and keep rule as
//              cogdl_b200_gat_fwd_dropout_f32), written only when a gradient is needed
//   mix[p,h] = (1 - alpha) * a * (dropped ? 0 : scale) + alpha * res[p,h]    (without res: a * (dropped ? 0 : scale))
// mix is what the layer aggregates (cogdl_b200_mhspmm_f32) and returns; no other [nnz, H] tensor is written.
//
// Backward (MODE 3 with the type term): given att and d mix (= mhsddmm(d out, h)),
//   d e[p,h]   = a * (g - sum_row a * g) * leakyrelu'(h_l[i,h] + h_r[j,h] + h_e[t,h]),  g = kept ? d mix * gscale : 0
//   g_row[i,h] = sum_{p in row i} d e[p,h]
// with gscale = (1 - alpha) / (1 - p_drop), in one pass.  The rest of the backward is existing code: the CSC
// mh-SpMM over mix for d h, edge_colsum for d h_r and the SpMM over the type-grouped slots for d h_e.
//
// The kernels and their launch plan are edge_softmax.cuh's, launched with TYPED (and MIX when res is given).
// h_e [T, H] is staged in a static shared-memory table of HGN_MAX_TABLE floats per block (4 KB: no kernel loses
// occupancy to it); larger tables are rejected before any launch.
#include "edge_softmax.cuh"

namespace cogdl_b200 {

static int hgn_check(int64_t n_rows, int64_t H, int64_t T, const char *who) {
  CB_REQUIRE(n_rows >= 0 && H >= 0, "%s: negative size", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && H < 0x7fffffffLL, "%s: sizes must fit int32", who);
  CB_REQUIRE(T >= 1 && T * H <= HGN_MAX_TABLE, "%s: the type table is [T=%lld, H=%lld]; T * H must be in [1, %d]", who,
             (long long)T, (long long)H, HGN_MAX_TABLE);
  return COGDL_B200_OK;
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_hgn_max_table(void) { return HGN_MAX_TABLE; }

extern "C" int cogdl_b200_hgn_attn_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *etype,
                                       const float *h_l, const float *h_r, const float *h_e, int64_t T,
                                       float negative_slope, uint64_t seed, uint64_t drop_below, float scale,
                                       const float *res_attn, float alpha, float *att_out, float *mix_out,
                                       int64_t n_rows, int64_t H, const cogdl_b200_hub_plan_t *plan,
                                       cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_hgn_attn_f32";
  int rc = hgn_check(n_rows, H, T, who);
  if (rc) return rc;
  CB_REQUIRE(isfinite(scale) && scale > 0.f, "%s: scale must be finite and > 0 (got %g)", who, (double)scale);
  CB_REQUIRE(isfinite(alpha), "%s: alpha must be finite (got %g)", who, (double)alpha);
  if (n_rows == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && etype && h_l && h_r && h_e && mix_out, "%s: null pointer", who);
  EsParams p;
  p.rowptr = rowptr; p.a = h_l; p.b = h_r; p.out = att_out; p.n_rows = n_rows; p.H = (int)H;
  p.colind = colind; p.slope = negative_slope; p.seed = seed; p.drop_below = drop_below;
  p.etype = etype; p.he = h_e; p.n_table = (int)(T * H); p.mix = mix_out; p.res = res_attn;
  p.alpha = alpha; p.keep = 1.f - alpha; p.keep_scale = scale;
  cudaStream_t s = (cudaStream_t)stream;
  const bool drop = drop_below > 0, mix = res_attn != nullptr;
  if (drop)
    return mix ? es_launch<2, true, true, true>(p, plan, s, who) : es_launch<2, true, true, false>(p, plan, s, who);
  return mix ? es_launch<2, false, true, true>(p, plan, s, who) : es_launch<2, false, true, false>(p, plan, s, who);
}

extern "C" int cogdl_b200_hgn_attn_bwd_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *etype,
                                           const float *att, const float *d_mix, const float *h_l, const float *h_r,
                                           const float *h_e, int64_t T, float negative_slope, float grad_scale,
                                           float *d_edge, float *g_row, int64_t n_rows, int64_t H,
                                           const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_hgn_attn_bwd_f32";
  int rc = hgn_check(n_rows, H, T, who);
  if (rc) return rc;
  CB_REQUIRE(isfinite(grad_scale), "%s: grad_scale must be finite (got %g)", who, (double)grad_scale);
  if (n_rows == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && etype && att && d_mix && h_l && h_r && h_e && d_edge && g_row, "%s: null pointer", who);
  EsParams p;
  p.rowptr = rowptr; p.a = att; p.b = d_mix; p.out = d_edge; p.n_rows = n_rows; p.H = (int)H;
  p.colind = colind; p.slope = negative_slope; p.hl = h_l; p.hr = h_r; p.grow = g_row; p.scale = grad_scale;
  p.etype = etype; p.he = h_e; p.n_table = (int)(T * H);
  return es_launch<3, true, true, false>(p, plan, (cudaStream_t)stream, who);
}

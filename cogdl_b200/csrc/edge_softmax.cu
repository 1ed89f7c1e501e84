// edge_softmax.cu -- per-destination-row softmax over edge logits [nnz, H]: forward, backward, the GAT
// attention form (logits computed on the fly) and the GAT attention backward, for sm_90a.
//
// Replaces edge_softmax / edge_softmax_backward (cogdl/operators/edge_softmax/edge_softmax.cu:7-98:
// one block of 32 x H threads per row, three passes over the row with lanes striding H floats apart
// -- <= 1/H sector efficiency -- and exp() evaluated twice) and, in MODE 2 / 3, the
// `leakyrelu(h_l[row] + h_r[col])` gathers + LeakyReLU + edge_softmax chain of
// cogdl/layers/gat_layer.py:73-74 and its autograd backward.  The kernels and their launch plan live in
// edge_softmax.cuh, which simple_hgn.cu launches with Simple-HGN's edge-type term and residual attention.
//
// Key layout fact: in CSR order the [deg, H] logits of row i are ONE contiguous block of deg*H floats
// at rowptr[i]*H, and consecutive rows are consecutive blocks.  With H a power of two <= 32, the
// element at offset t has head t % H, so a thread striding by a multiple of H keeps its head and
// per-head reductions are xor-shuffles over lane strides 16 .. H.
//
// Work decomposition with a hub plan (round 2; one or two launches on the caller's stream, no side
// stream, no events, no cluster kernel):
//   items = SEGMENTS (runs of consecutive non-hub rows, ~seg_cost rows+edges) and hub CHUNKS (<= chunk_edges
//   edges of one hub row), one warp per item -- the same items as the row-stream SpMM.
//   * es_stats_kernel (only when the graph has hub rows): every chunk reduces its own (max, sum exp)
//     per head; the last chunk of a row to arrive merges them IN CHUNK ORDER into the row's (M, S)
//     (deterministic; a 22 K-edge hub is reduced by 350 warps on many SMs instead of serialising on
//     one SM, and nobody spins waiting for anybody).
//   * es_main_kernel (launched as a PROGRAMMATIC DEPENDENT of the statistics kernel: it starts while that one is
//     still running; segments come first in its grid and need nothing from it, chunk items come last and execute
//     griddepcontrol.wait): a chunk normalises its elements with its row's (M, S); a segment stages whole
//     rows in shared memory -- by ONE `cp.async.bulk` (TMA 1-D, UBLKCP) per window completed on an
//     mbarrier when the tile is 16-byte aligned, else by coalesced loads --, computes max / sum exp /
//     normalise per (row, head) pair held by one lane, and writes the tile back with one bulk store.
//     Rows of a window are visited in DEGREE-SORTED order (one 32-key bitonic sort in registers), so the
//     32/H rows a warp works on at a time have near-equal trip counts: on power-law rows (median 3
//     edges, tail to 64) this is what removes the lane divergence that dominated round 1's kernel.
//     (A register-resident variant -- every lane owning coalesced elements, two-level per-(row, head) folds, no
//     staging, ~3x fewer instructions -- was built, validated and measured slower: only 24 warps/SM of 2 KB
//     windows leave each window's latency chain exposed.  Removed.)
// Without a plan every row takes the warp path (es_warp_kernel); head counts that are not a power of
// two, or > 32, use a generic strided kernel.
//   MODE 0: forward, a = logits        MODE 1: backward, a = y, b = g  -> y * (g - sum_row y*g)
//   MODE 2: attention, a = h_l [N,H], b = h_r [N,H]: logit = leakyrelu(a[row,h] + b[col,h])
//   MODE 3: attention backward: y = att, g = d att (from mhsddmm), plus h_l / h_r / colind / slope:
//           out = d logit * leakyrelu'(h_l[row]+h_r[col]) written to [nnz,H], and grow[row,h] = its row sum
// DROP (template flag of MODES 2 and 3, attention dropout): (edge p, head h) is dropped iff draw(seed, p, h) <
// drop_below (rng.cuh; p = CSR position, so the CSC backward finds the same mask through perm).  MODE 2 writes a
// dropped attention as -a: the softmax is >= 0, so its sign bit is free to carry the mask, and the hash runs once per
// (edge, head) here instead of in the gather loops.  MODE 3 reads y = |att| and g = (sign bit ? 0 : d att * scale),
// the gradient of the softmax before the dropout.  The bit is tested, never `att < 0`: a dropped softmax that
// underflowed to 0 is -0.0.
#include "edge_softmax.cuh"

namespace cogdl_b200 {

template <int MODE>
static int es_entry(const int32_t *rowptr, const float *a, const float *b, float *out, int64_t n_rows,
                    int64_t H, const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream,
                    const char *who) {
  CB_REQUIRE(n_rows >= 0 && H >= 0, "%s: negative size", who);
  if (n_rows == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && a && out && (MODE != 1 || b), "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && H < 0x7fffffffLL, "%s: sizes must fit int32", who);
  EsParams p;
  p.rowptr = rowptr; p.a = a; p.b = b; p.out = out; p.n_rows = n_rows; p.H = (int)H;
  return es_launch<MODE, false, false, false>(p, plan, (cudaStream_t)stream, who);
}

// GAT attention (used by cogdl_b200_gat_fwd_f32 / _dropout_f32, mhspmm.cu): att = softmax_row(leakyrelu(h_l[row] +
// h_r[col])), any H; with drop, the dropped (edge, head) pairs carry the sign bit.
int gat_attention(const int32_t *rowptr, const int32_t *colind, const float *h_l, const float *h_r, float slope,
                  float *att, int64_t n_rows, int64_t H, const cogdl_b200_hub_plan_t *plan, cudaStream_t s,
                  bool drop, uint64_t seed, uint64_t drop_below) {
  EsParams p;
  p.rowptr = rowptr; p.a = h_l; p.b = h_r; p.out = att; p.n_rows = n_rows; p.H = (int)H;
  p.colind = colind; p.slope = slope; p.seed = seed; p.drop_below = drop_below;
  if (drop) return es_launch<2, true, false, false>(p, plan, s, "cogdl_b200_gat_fwd_dropout_f32");
  return es_launch<2, false, false, false>(p, plan, s, "cogdl_b200_gat_fwd_f32");
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_edge_softmax_scratch_bytes(int64_t n_chunks, int64_t H) {
  return n_chunks * H * (int64_t)(sizeof(float2) + sizeof(float));
}

extern "C" int cogdl_b200_edge_softmax_fwd_f32(const int32_t *rowptr, const float *in, float *out,
                                               int64_t n_rows, int64_t H,
                                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return es_entry<0>(rowptr, in, nullptr, out, n_rows, H, plan, stream, "cogdl_b200_edge_softmax_fwd_f32");
}

extern "C" int cogdl_b200_edge_softmax_bwd_f32(const int32_t *rowptr, const float *y, const float *g,
                                               float *gin, int64_t n_rows, int64_t H,
                                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return es_entry<1>(rowptr, y, g, gin, n_rows, H, plan, stream, "cogdl_b200_edge_softmax_bwd_f32");
}

// GAT attention backward: given att = softmax_row(leakyrelu(h_l[row] + h_r[col])) and d att (= mhsddmm(d out, feat)):
//   d e[p,h]  = att * (d att - sum_row att * d att) * leakyrelu'(h_l[row,h] + h_r[col,h])      -> d_edge [nnz, H]
//   g_row[i,h] = sum_{p in row i} d e[p,h]                                                      -> [n_rows, H]
// (g_col is the column-wise sum of d_edge: cogdl_b200_edge_colsum_f32 on the cached transpose.)
template <bool DROP>
static int gat_attn_bwd(const int32_t *rowptr, const int32_t *colind, const float *att, const float *d_att,
                        const float *h_l, const float *h_r, float negative_slope, float scale, float *d_edge,
                        float *g_row, int64_t n_rows, int64_t H, const cogdl_b200_hub_plan_t *plan,
                        cogdl_b200_stream_t stream, const char *who) {
  CB_REQUIRE(n_rows >= 0 && H >= 0, "%s: negative size", who);
  if (n_rows == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && att && d_att && h_l && h_r && d_edge && g_row, "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && H < 0x7fffffffLL, "%s: sizes must fit int32", who);
  EsParams p;
  p.rowptr = rowptr; p.a = att; p.b = d_att; p.out = d_edge; p.n_rows = n_rows; p.H = (int)H;
  p.colind = colind; p.slope = negative_slope; p.hl = h_l; p.hr = h_r; p.grow = g_row; p.scale = scale;
  return es_launch<3, DROP, false, false>(p, plan, (cudaStream_t)stream, who);
}

extern "C" int cogdl_b200_gat_attn_bwd_f32(const int32_t *rowptr, const int32_t *colind, const float *att,
                                           const float *d_att, const float *h_l, const float *h_r,
                                           float negative_slope, float *d_edge, float *g_row, int64_t n_rows,
                                           int64_t H, const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return gat_attn_bwd<false>(rowptr, colind, att, d_att, h_l, h_r, negative_slope, 1.f, d_edge, g_row, n_rows, H, plan,
                             stream, "cogdl_b200_gat_attn_bwd_f32");
}

// The same over the signed attention of cogdl_b200_gat_fwd_dropout_f32: d_att (= mhsddmm(d out, feat)) is the
// gradient of the dropped, scaled attention; the softmax backward runs on |att| with d_att * scale on the kept
// entries and 0 on the dropped ones.
extern "C" int cogdl_b200_gat_attn_bwd_dropout_f32(const int32_t *rowptr, const int32_t *colind, const float *att,
                                                   const float *d_att, const float *h_l, const float *h_r,
                                                   float negative_slope, float scale, float *d_edge, float *g_row,
                                                   int64_t n_rows, int64_t H, const cogdl_b200_hub_plan_t *plan,
                                                   cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_gat_attn_bwd_dropout_f32";
  CB_REQUIRE(isfinite(scale) && scale > 0.f, "%s: scale must be finite and > 0 (got %g)", who, (double)scale);
  return gat_attn_bwd<true>(rowptr, colind, att, d_att, h_l, h_r, negative_slope, scale, d_edge, g_row, n_rows, H,
                            plan, stream, who);
}

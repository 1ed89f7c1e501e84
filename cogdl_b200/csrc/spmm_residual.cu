// spmm_residual.cu -- the fp32 SpMM with a residual epilogue (GCNII / APPNP initial-residual propagation), sm_90a.
//
//   Y[i,:] = fl( fl(a * fl(r[i] * (A @ X)[i,:])) + fl(b * Z[i,:]) )        r and Z optional
//
// The propagation step of GCNII (cogdl/layers/gcnii_layer.py:24-30) and APPNP (cogdl/models/nn/ppnp.py:77-83) is
// `(1 - alpha) * spmm(graph, x) + alpha * init_x`, with the graph's in_norm applied after the SpMM: four eager passes
// over [N, F] after the aggregation.  Every store site of the SpMM already holds the finished row, so the epilogue is
// applied there: the row kernel's row and hub-merge stores, the row-stream loops' row ends (general, lean one-pass and
// lean panel), their hub merge and the empty-row zero fill (an empty row is the epilogue of a zero sum).  A (A @ X)
// is the plain SpMM's, in its accumulation order, and each epilogue step is one fp32 multiply or add in the unfused
// sequence's order, so Y is bit-identical to that sequence.  The kernels and their dispatch are the SpMM's (spmm.cuh,
// stream.cuh) with RESID set; this file holds their instantiations and the entry point.
#include "spmm.cuh"

namespace cogdl_b200 {

// [p, p + n) and [q, q + m) share a byte
static bool overlaps(const float *p, int64_t n, const float *q, int64_t m) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
  return a < b + (uintptr_t)m * sizeof(float) && b < a + (uintptr_t)n * sizeof(float);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int cogdl_b200_spmm_residual_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                                            const float *X, int64_t x_rows, const float *Z, float a, float b,
                                            const float *row_scale, float *Y, int64_t n_rows, int64_t F,
                                            int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                            cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_spmm_residual_f32";
  CB_REQUIRE(n_rows >= 0 && F >= 0, "%s: negative size (n_rows=%lld, F=%lld)", who, (long long)n_rows, (long long)F);
  CB_REQUIRE(x_rows >= 0 && panels >= 0, "%s: negative x_rows / panels", who);
  if (n_rows == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && X && Y, "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "%s: n_rows / F must fit int32", who);
  // the kernels read X, Z and row_scale (read-only cache path) while other warps write finished Y rows; X holds
  // x_rows rows (colind < x_rows), so an empty X can only coincide with Y
  CB_REQUIRE(Y != X && !overlaps(Y, n_rows * F, X, x_rows * F), "%s: Y overlaps X", who);
  CB_REQUIRE(!Z || !overlaps(Y, n_rows * F, Z, n_rows * F), "%s: Y overlaps Z", who);
  CB_REQUIRE(!row_scale || !overlaps(Y, n_rows * F, row_scale, n_rows), "%s: Y overlaps row_scale", who);
  int rc = check_plan(plan, (plan ? (int64_t)plan->n_chunks : 0) * F * (int64_t)sizeof(float));
  if (rc) return rc;
  SpmmParams p;
  p.rowptr = rowptr; p.colind = colind; p.val = val; p.X0 = X; p.X1 = X; p.n0 = INT64_MAX;
  p.Y = Y; p.n_rows = n_rows; p.hub = hub_view(plan);
  p.n_peers = 0; p.peer_shift = 0;
  for (int i = 0; i < 8; ++i) p.peers[i] = nullptr;
  p.Z = Z; p.row_scale = row_scale; p.res_a = a; p.res_b = b;
  const bool vec = (F % 4 == 0) && aligned16(X) && aligned16(Y) && aligned16(Z) &&
                   (p.hub.n_chunks == 0 || aligned16(p.hub.partials));
  if (vec) p.FV = (int)(F / 4);
  const bool panel_form = vec && p.hub.n_segs > 0 && F % 32 == 0;
  if (panels > 1)
    CB_REQUIRE(panel_form && panel_width_ok(F, panels),
               "%s: %d panels need a plan with segments, 16-byte aligned buffers and F / panels in {32, 64, 128} "
               "(F=%lld, at most %d panels)", who, panels, (long long)F, COGDL_B200_MAX_PANELS);
  const int P = panels == 0 ? (panel_form ? auto_panels(x_rows, F) : 1) : panels;
  if (P > 1) return launch_spmm_panels<true>(p, F, P, (cudaStream_t)stream);
  if (vec) return dispatch_spmm<float4, true>(p, (cudaStream_t)stream);
  p.FV = (int)F;
  return dispatch_spmm<float, true>(p, (cudaStream_t)stream);
}

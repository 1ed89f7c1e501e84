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
// stream.cuh) with EPI_RESID; this file holds their instantiations and the entry point.
#include "spmm.cuh"

using namespace cogdl_b200;

extern "C" int cogdl_b200_spmm_residual_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                                            const float *X, int64_t x_rows, const float *Z, float a, float b,
                                            const float *row_scale, float *Y, int64_t n_rows, int64_t F,
                                            int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                            cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_spmm_residual_f32";
  // the kernels read X, Z and row_scale (read-only cache path) while other warps write finished Y rows; X holds
  // x_rows rows (colind < x_rows), so an empty X can only coincide with Y.  An empty Y is written by no one.
  if (n_rows > 0 && F > 0) {
    CB_REQUIRE(Y != X && !overlaps(Y, n_rows * F, X, x_rows * F), "%s: Y overlaps X", who);
    CB_REQUIRE(!Z || !overlaps(Y, n_rows * F, Z, n_rows * F), "%s: Y overlaps Z", who);
    CB_REQUIRE(!row_scale || !overlaps(Y, n_rows * F, row_scale, n_rows), "%s: Y overlaps row_scale", who);
  }
  return spmm_entry<EPI_RESID>(rowptr, colind, val, X, INT64_MAX, nullptr, Y, n_rows, F, plan, stream, who, nullptr, 0, 0,
                          x_rows, panels, Z, row_scale, a, b);
}

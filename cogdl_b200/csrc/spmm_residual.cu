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
// sequence's order, so Y is bit-identical to that sequence.  The kernels and their dispatch are the SpMM's: the row and
// row-stream kernels (spmm.cuh, stream.cuh) with EPI = EPI_RESID, only that form instantiated here, behind the entry
// point.
#include "spmm.cuh"

using namespace cogdl_b200;

extern "C" int cogdl_b200_spmm_residual_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                                            const float *X, int64_t x_rows, const float *Z, float a, float b,
                                            const float *row_scale, float *Y, int64_t n_rows, int64_t F,
                                            int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                            cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_spmm_residual_f32";
  if (n_rows > 0 && F > 0) {     // an empty Y is written by no one
    const int rc = check_output_apart(who, "Y", Y, n_rows, F, X, x_rows, Z, row_scale);
    if (rc) return rc;
  }
  SpmmEpilogue epi;
  epi.Z = Z; epi.row_scale = row_scale; epi.res_a = a; epi.res_b = b;
  return spmm_entry<EPI_RESID>(rowptr, colind, val, X, INT64_MAX, nullptr, Y, n_rows, F, plan, stream, who, nullptr, 0, 0,
                               x_rows, panels, epi);
}

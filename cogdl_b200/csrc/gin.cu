// gin.cu -- the fp32 SpMM with a residual epilogue whose coefficient is read on the device (GIN / GINE), sm_90a.
//
//   Y[i,:] = fl( fl(a * fl(r[i] * (A @ X)[i,:])) + fl((*b_dev) * Z[i,:]) )        r and Z optional
//
// GIN's aggregation (cogdl/layers/gin_layer.py:35, gine_layer.py:33-34) is `(1 + eps) * x + spmm(graph, x)`, with eps
// a trainable one-element parameter on the device: one SpMM and three eager passes over [N, F].  The residual
// epilogue (spmm_residual.cu) computes it with a = 1 and b = fl(1 + eps), but takes b as a host float, which would cost
// a host synchronisation per layer to read eps.  Here b is read by the kernel from b_dev, so the launch is queued
// behind whatever computes 1 + eps without the host waiting.  Rounding and store sites are the residual epilogue's
// (fp32 addition commutes, so with a = 1 the forward is bit-identical to the reference expression on this package's
// spmm); the backward's d x = A^T (r g) + (1 + eps) g is the same launch over the adjoint.  The kernels and their
// dispatch are the SpMM's: the row and row-stream kernels (spmm.cuh, stream.cuh) with EPI = EPI_RESID_DEV, only that
// form instantiated here, behind the entry point.
#include "spmm.cuh"

using namespace cogdl_b200;

extern "C" int cogdl_b200_spmm_residual_dcoef_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                                                  const float *X, int64_t x_rows, const float *Z, float a,
                                                  const float *b_dev, const float *row_scale, float *Y, int64_t n_rows,
                                                  int64_t F, int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                                  cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_spmm_residual_dcoef_f32";
  // b_dev is read (read-only cache path) as X, Z and row_scale are, so Y may not overlap it either.  The coefficient
  // multiplies Z, so Z needs it.
  if (n_rows > 0 && F > 0) {
    const int rc = check_output_apart(who, "Y", Y, n_rows, F, X, x_rows, Z, row_scale);
    if (rc) return rc;
    CB_REQUIRE(!Z || b_dev, "%s: Z needs the coefficient b_dev", who);
    CB_REQUIRE(!b_dev || !overlaps(Y, n_rows * F, b_dev, 1), "%s: Y overlaps b_dev", who);
  }
  SpmmEpilogue epi;
  epi.Z = Z; epi.row_scale = row_scale; epi.res_a = a; epi.res_b_dev = b_dev;
  return spmm_entry<EPI_RESID_DEV>(rowptr, colind, val, X, INT64_MAX, nullptr, Y, n_rows, F, plan, stream, who, nullptr,
                                   0, 0, x_rows, panels, epi);
}

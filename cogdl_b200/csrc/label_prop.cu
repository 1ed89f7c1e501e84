// label_prop.cu -- one label-propagation step of Correct & Smooth in one SpMM launch, sm_90a.
//
//   Y[i,:] = pin[i] ? Z[i,:]
//                   : clamp( fl( fl(a * fl(r[i] * (A @ X)[i,:])) + fl(b * Z[i,:]) ), lo, hi )      r, Z, pin, clamp optional
//
// The loop of Correct & Smooth (cogdl/models/nn/correct_smooth.py, outcome_correlation) is
// `result = alpha * spmm(g, result); result += (1 - alpha) * labels; result = post_step(result)`, with post_step either
// torch.clamp(result, lower, upper) (autoscale_post) or `result[nid] = labels[nid]` (fixed_post): one SpMM and four or
// five eager passes over [N, C] per iteration.  The residual epilogue (spmm_residual.cu) already gives the first two
// lines bit for bit at every store site of the SpMM; this epilogue adds the post step there.  The clamp is the
// expression torch's CUDA clamp evaluates (a NaN passes, else fminf(fmaxf(v, lo), hi)), so it rounds nothing and
// matches torch for -0.0 and lo > hi.  A pinned row stores Z's row bit for bit, whatever its sum, which is what the
// row reset leaves behind.  The store sites are the residual epilogue's: the row kernel's row and hub-merge stores,
// the row-stream loops' row ends (general, lean one-pass and lean panel), their hub merge and the empty-row fill.  The
// kernels and their dispatch are the SpMM's (spmm.cuh, stream.cuh) with EPI_LABELPROP; this file holds their
// instantiations and the entry point.
#include "spmm.cuh"

using namespace cogdl_b200;

extern "C" int cogdl_b200_label_prop_f32(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X,
                                         int64_t x_rows, const float *Z, float a, float b, const float *row_scale,
                                         const uint8_t *pin, int32_t has_clamp, float lo, float hi, float *Y,
                                         int64_t n_rows, int64_t F, int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                         cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_label_prop_f32";
  // as cogdl_b200_spmm_residual_f32: X, Z and row_scale are read (read-only cache path) while finished Y rows are
  // written, so Y may overlap none of them.  A pinned row is Z's row, so pin needs Z.
  if (n_rows > 0 && F > 0) {
    CB_REQUIRE(Y != X && !overlaps(Y, n_rows * F, X, x_rows * F), "%s: Y overlaps X", who);
    CB_REQUIRE(!Z || !overlaps(Y, n_rows * F, Z, n_rows * F), "%s: Y overlaps Z", who);
    CB_REQUIRE(!row_scale || !overlaps(Y, n_rows * F, row_scale, n_rows), "%s: Y overlaps row_scale", who);
    CB_REQUIRE(!pin || Z, "%s: pinned rows need Z", who);
  }
  return spmm_entry<EPI_LABELPROP>(rowptr, colind, val, X, INT64_MAX, nullptr, Y, n_rows, F, plan, stream, who, nullptr,
                                   0, 0, x_rows, panels, Z, row_scale, a, b, pin, has_clamp != 0, lo, hi);
}

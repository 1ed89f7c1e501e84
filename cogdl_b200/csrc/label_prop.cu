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
// kernels and their dispatch are the SpMM's: the row and row-stream kernels (spmm.cuh, stream.cuh) with
// EPI = EPI_LABELPROP, only that form instantiated here, behind the entry point.
#include "spmm.cuh"

using namespace cogdl_b200;

extern "C" int cogdl_b200_label_prop_f32(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X,
                                         int64_t x_rows, const float *Z, float a, float b, const float *row_scale,
                                         const uint8_t *pin, int32_t has_clamp, float lo, float hi, float *Y,
                                         int64_t n_rows, int64_t F, int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                         cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_label_prop_f32";
  // a pinned row is Z's row, so pin needs Z
  if (n_rows > 0 && F > 0) {
    const int rc = check_output_apart(who, "Y", Y, n_rows, F, X, x_rows, Z, row_scale);
    if (rc) return rc;
    CB_REQUIRE(!pin || Z, "%s: pinned rows need Z", who);
  }
  SpmmEpilogue epi;
  epi.Z = Z; epi.row_scale = row_scale; epi.res_a = a; epi.res_b = b;
  epi.pin = pin; epi.has_clamp = has_clamp != 0; epi.clamp_lo = lo; epi.clamp_hi = hi;
  return spmm_entry<EPI_LABELPROP>(rowptr, colind, val, X, INT64_MAX, nullptr, Y, n_rows, F, plan, stream, who, nullptr,
                                   0, 0, x_rows, panels, epi);
}

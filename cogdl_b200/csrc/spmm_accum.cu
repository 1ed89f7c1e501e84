// spmm_accum.cu -- one hop of GRAND's random propagation in one SpMM launch, sm_90a.
//
//   Xn[i,:]  = fl(r[i] * (A @ X)[i,:])                                  stored unless this is the last hop
//   ACC[i,:] = fl(ACC_in[i,:] + Xn[i,:]),  then fl(ACC[i,:] * scale) on the last hop
//
// GRAND's propagation (cogdl/models/nn/grand.py:98-104) is, after DropNode, `y = x; for i in range(order):
// x = spmm(graph, x); y.add_(x)` and then `y.div_(order + 1.0)`: per hop one SpMM (with the graph's in_norm) and one
// read-modify-write pass of y, and one more pass at the end.  Here the add and, on the last hop, the scaling run in
// the SpMM's store: each finished row is stored as the hop's output and added to the running sum ACC in the same
// store site.  On CUDA `y.div_(s)` with a host scalar s multiplies by the fp32 reciprocal 1 / s (torch's div_true
// kernel), so the caller passes scale = fl(1 / (order + 1)) and the result is bit-identical to the reference loop on
// this package's spmm.  ACC is never gathered in the launch that writes it, so its in-place read and write of the same
// element by the same thread are race-free; ACC_in (NULL: ACC itself) lets the first hop read the hop-0 features
// without a copy.  The store sites are the residual epilogue's: the row kernel's row and hub-merge stores, the
// row-stream loops' row ends (general, lean one-pass and lean panel), their hub merge and the empty-row fill.  The
// kernels and their dispatch are the SpMM's: the row and row-stream kernels (spmm.cuh, stream.cuh) with
// EPI = EPI_ACCUM, only that form instantiated here, behind the entry point.
#include "spmm.cuh"

using namespace cogdl_b200;

extern "C" int cogdl_b200_spmm_accum_f32(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X,
                                         int64_t x_rows, const float *row_scale, const float *acc_in, float *acc,
                                         int32_t last, float scale, float *Xn, int64_t n_rows, int64_t F,
                                         int32_t panels, const cogdl_b200_hub_plan_t *plan,
                                         cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_spmm_accum_f32";
  const float *in = acc_in ? acc_in : acc;
  // Neither output, Xn nor ACC, may overlap X or row_scale, nor each other.  ACC_in is read by the thread that writes
  // the same element of ACC: it is ACC itself or lies apart from it.
  if (n_rows > 0 && F > 0) {
    const int64_t nf = n_rows * F;
    CB_REQUIRE(acc, "%s: null ACC", who);
    CB_REQUIRE(last || Xn, "%s: Xn may be NULL on the last hop only", who);
    int rc = check_output_apart(who, "ACC", acc, n_rows, F, X, x_rows, nullptr, row_scale);
    if (rc) return rc;
    CB_REQUIRE(in == acc || !overlaps(acc, nf, in, nf), "%s: ACC_in overlaps ACC without being it", who);
    if (!last) {
      rc = check_output_apart(who, "Xn", Xn, n_rows, F, X, x_rows, nullptr, row_scale);
      if (rc) return rc;
      CB_REQUIRE(!overlaps(Xn, nf, acc, nf), "%s: Xn overlaps ACC", who);
      CB_REQUIRE(!overlaps(Xn, nf, in, nf), "%s: Xn overlaps ACC_in", who);
    }
  }
  SpmmEpilogue epi;
  epi.Z = in; epi.row_scale = row_scale; epi.acc = acc; epi.acc_last = last != 0; epi.acc_scale = scale;
  // on the last hop nothing but ACC is written: it stands in as Y, the base the store sites index from
  return spmm_entry<EPI_ACCUM>(rowptr, colind, val, X, INT64_MAX, nullptr, last ? acc : Xn, n_rows, F, plan, stream, who,
                               nullptr, 0, 0, x_rows, panels, epi);
}

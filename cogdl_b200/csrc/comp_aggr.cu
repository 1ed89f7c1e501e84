// comp_aggr.cu -- CompGCN composition aggregation for sm_90a.
//
//   Y[i,:] = sum_{q in row i} w[q] * phi(A[colind[q],:], B[idx2[q],:])     phi = a * b | a - b | a
//
// Replaces the message passing of CompGCNLayer (cogdl/models/nn/compgcn.py:124-140), which gathers x[col] and
// rel_embed[type] into [E/2, F_in] tensors, composes them, multiplies the per-edge result by W ([E/2, F_out]),
// scales it by the edge norm and scatter_adds it with float atomics.  The message is linear in W, so the layer
// only needs this aggregation (output [rows, F_in]) followed by N-row GEMMs.  One kernel family serves the
// three passes of the layer (the caller picks the structure):
//   forward  rows = the two edge halves stacked (2N rows), A = x by column, B = R' by edge type;
//   dx       rows = the transpose of that 2N x N matrix, A = dagg by stacked row, B = R' by edge type (mult)
//            or phi = a (sub);
//   dR'      rows = edge types, A = dagg by stacked row, B = x by column (mult) or phi = a (sub, negated by
//            the caller).
// The loop is the row-stream skeleton (stream.cuh) with a second int32 index per slot and a second gathered
// row: the relation table is small and stays in the L2, so an edge costs one more 4-byte index and one more
// L2 hit than the SpMM.  Hub rows are cut into the plan's chunks and merged in chunk order (no atomics):
// results are bit-reproducible.
#include "common.cuh"
#include "stream.cuh"

namespace cogdl_b200 {

template <typename VecT, int NV, int MODE>
static int launch_comp(const StreamParams &p, cudaStream_t stream) {
  // U gathers of two rows each in flight per lane: the same bytes in flight as the SpMM's U, twice the registers
  constexpr int U = (NV == 1) ? 4 : 2;
  const int64_t warps = (int64_t)p.hub.n_chunks + p.hub.n_segs;
  const int64_t blocks = ceil_div(warps * 32, STREAM_BLOCK);
  if (blocks == 0) return COGDL_B200_OK;
  if (blocks > 0x7fffffffLL) return set_error(COGDL_B200_EINVAL, "cogdl_b200_comp_aggr_f32: problem too large for one launch");
  note_kernel("cogdl_b200::stream_kernel<%s,NV=%d,%s,SRC_ONE,U=%d,MINB=1,prefetch> block=%d",
              sizeof(VecT) == 16 ? "float4" : "float", NV,
              MODE == MODE_COMP_MULT ? "comp_mult" : (MODE == MODE_COMP_SUB ? "comp_sub" : "weighted"), U,
              STREAM_BLOCK);
  stream_kernel<VecT, NV, MODE, false, SRC_ONE, U, 1, true><<<(unsigned)blocks, STREAM_BLOCK, 0, stream>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

template <typename VecT, int MODE>
static int dispatch_comp(const StreamParams &p, cudaStream_t s) {
  // one vector per lane up to 32 vectors, two beyond (rows wider than 64 vectors loop over column tiles)
  if (p.ldv <= 32) return launch_comp<VecT, 1, MODE>(p, s);
  return launch_comp<VecT, 2, MODE>(p, s);
}

template <typename VecT>
static int dispatch_op(const StreamParams &p, int op, cudaStream_t s) {
  if (op == COGDL_B200_COMP_MULT) return dispatch_comp<VecT, MODE_COMP_MULT>(p, s);
  if (op == COGDL_B200_COMP_SUB) return dispatch_comp<VecT, MODE_COMP_SUB>(p, s);
  return dispatch_comp<VecT, MODE_WEIGHTED>(p, s);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int64_t cogdl_b200_comp_aggr_scratch_bytes(int64_t n_chunks, int64_t F) {
  return n_chunks > 0 && F > 0 ? n_chunks * F * (int64_t)sizeof(float) : 0;
}

extern "C" int cogdl_b200_comp_aggr_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *idx2,
                                        const float *w, const float *A, int64_t a_rows, const float *B,
                                        int64_t b_rows, float *Y, int64_t n_rows, int64_t F, int32_t op,
                                        const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  const char *who = "cogdl_b200_comp_aggr_f32";
  CB_REQUIRE(op == COGDL_B200_COMP_MULT || op == COGDL_B200_COMP_SUB || op == COGDL_B200_COMP_COPY,
             "%s: unknown op %d (mult = %d, sub = %d, copy = %d)", who, op, COGDL_B200_COMP_MULT, COGDL_B200_COMP_SUB,
             COGDL_B200_COMP_COPY);
  CB_REQUIRE(F > 0 && F < 0x7fffffffLL, "%s: F must be in [1, 2^31), got %lld", who, (long long)F);
  CB_REQUIRE(n_rows >= 0 && n_rows < 0x7fffffffLL && a_rows >= 0 && b_rows >= 0, "%s: bad row count", who);
  if (n_rows == 0) return COGDL_B200_OK;
  const bool two = op != COGDL_B200_COMP_COPY;
  CB_REQUIRE(rowptr && colind && w && A && Y && (!two || (idx2 && B)), "%s: null pointer", who);
  CB_REQUIRE(a_rows > 0 && (!two || b_rows > 0), "%s: empty source table (a_rows=%lld, b_rows=%lld)", who,
             (long long)a_rows, (long long)b_rows);
  CB_REQUIRE(plan && plan->chunk_edges > 0, "%s: needs a hub plan", who);
  CB_REQUIRE(plan->n_hub_rows <= n_rows && (plan->n_segs > 0 || plan->n_hub_rows == n_rows),
             "%s: the plan does not match the structure's %lld rows (%d hub rows, %d segments)", who,
             (long long)n_rows, plan->n_hub_rows, plan->n_segs);
  int rc = check_plan(plan, cogdl_b200_comp_aggr_scratch_bytes(plan->n_chunks, F));
  if (rc) return rc;
  StreamParams p = {};
  p.rowptr = rowptr; p.colind = colind; p.val = w; p.idx2 = two ? idx2 : nullptr; p.B = two ? B : nullptr;
  p.X0 = A; p.X1 = A; p.n0 = INT64_MAX; p.Y = Y; p.H = 1; p.S = 1;
  p.hub = hub_view(plan);
  const bool vec = (F % 4 == 0) && aligned16(A) && (!two || aligned16(B)) && aligned16(Y) &&
                   (p.hub.n_chunks == 0 || aligned16(p.hub.partials));
  p.ldv = p.FVL = (int)(vec ? F / 4 : F);
  if (vec) return dispatch_op<float4>(p, op, (cudaStream_t)stream);
  return dispatch_op<float>(p, op, (cudaStream_t)stream);
}

/*
 * cogdl_b200.h -- C ABI of libcogdl_b200.so: H100 (sm_90a) kernels for CogDL's sparse
 * message-passing hot path (CSR SpMM / SDDMM / edge-softmax / multi-head SpMM / scatter_max).
 *
 * This is the drop-in boundary.  Each entry point replaces one function that the reference
 * exposes today through a pybind11/torch extension (THUDM/CogDL @ 281f4742; paths relative to
 * the CogDL tree).  Differences from the reference ABI, all deliberate:
 *   - plain C: raw device pointers + int64 sizes + an opaque stream handle, no torch types;
 *   - the caller owns every buffer (outputs included); no device memory is allocated here (the
 *     reference leaks a cusparseHandle and cudaMalloc's per call, spmm_kernel.cu:517-531); the library
 *     keeps no streams or events of its own;
 *   - work is enqueued on the caller's stream (the reference uses the legacy default stream);
 *   - errors are returned (0 = ok, <0 = COGDL_B200_E*), text via cogdl_b200_last_error();
 *     the reference `assert`s / exit(1)s (spmm.cpp:28-39, computeUtil.h:13-27);
 *   - offsets are 64-bit (the reference overflows int32 at N*F >= 2^31, spmm_kernel.cu:393).
 * Index dtype is int32 and feature dtype fp32, exactly as the reference kernels take them
 * (`rowptr.int(), colind.int()`, cogdl/utils/spmm_utils.py:106).  All arrays are contiguous,
 * row-major; float arrays must be 4-byte aligned (16-byte alignment enables the vector path).
 *
 * No CPU fallback exists in this library: every call needs a CUDA device of compute
 * capability 10.x and fails with COGDL_B200_EDEVICE otherwise.
 */
#ifndef COGDL_B200_H_
#define COGDL_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COGDL_B200_ABI_VERSION 6

#define COGDL_B200_OK 0
#define COGDL_B200_EINVAL (-1)   /* bad argument (null pointer, negative size, unsupported shape) */
#define COGDL_B200_ECUDA (-2)    /* a CUDA runtime call or kernel launch failed */
#define COGDL_B200_EDEVICE (-3)  /* no sm_90 device / kernel image not loadable */
#define COGDL_B200_ESCRATCH (-4) /* hub-plan scratch too small for this call */

/* Exported-symbol marker (the library is built with -fvisibility=hidden). */
#if defined(COGDL_B200_BUILD)
#define COGDL_B200_API __attribute__((visibility("default")))
#else
#define COGDL_B200_API
#endif

/* cudaStream_t, passed as an opaque pointer (NULL = legacy default stream). */
typedef void *cogdl_b200_stream_t;

COGDL_B200_API int cogdl_b200_abi_version(void);
/* Thread-local text of the last error returned on this thread ("" if none). */
COGDL_B200_API const char *cogdl_b200_last_error(void);
/* 0 if the current device can run this library (compute capability 10.x), else EDEVICE. */
COGDL_B200_API int cogdl_b200_check_device(void);
/* Number of kernels this library has launched in this process (all threads). */
COGDL_B200_API int64_t cogdl_b200_launch_count(void);
/* Thread-local description of the kernel instantiation chosen by the last dispatching call on this
 * thread (e.g. "stream_kernel<float4,NV=1,weighted,SRC_ONE,U=4>"); "" before the first call.  Lets a
 * harness check that a profile it cites is of the kernel that actually ran. */
COGDL_B200_API const char *cogdl_b200_last_kernel(void);

/* ---------------------------------------------------------------------------------------
 * Hub plan: how rows with more than `chunk_edges` edges are cut into fixed-size edge chunks
 * so that a power-law hub does not serialise on one warp (the reference serialises it:
 * one warp per row, spmm_kernel.cu:370-440).  Built once per CSR structure, reused by every
 * op below; optional (plan == NULL => every row is processed whole, in CSR order).
 *
 *   hub_rows[n_hub_rows]        rows with degree > chunk_edges (any order)
 *   chunks[2*n_chunks]          (row, first_slot) per chunk slot; a row's chunks occupy the
 *                               contiguous slots [first_slot, first_slot + ceil(deg/chunk_edges))
 *                               and chunk j covers edges rowptr[row] + j*chunk_edges ...
 *   counters[n_chunks * COGDL_B200_MAX_PANELS]
 *                               zero on entry; left zero on exit (arrival counters; the panel form of
 *                               the SpMM keeps one set of n_chunks per column panel)
 *   partials                    scratch for per-chunk partial results; `partials_bytes` capacity.
 *                               Each entry point below names the cogdl_b200_*_scratch_bytes query
 *                               that gives its need (COGDL_B200_ESCRATCH when it is not met).
 * counters/partials are per-stream scratch: do not share one plan between concurrent streams.
 * Partial results of a hub row are combined in chunk order by the last chunk to finish, so
 * results are deterministic run to run.
 * ------------------------------------------------------------------------------------- */
#define COGDL_B200_MAX_PANELS 8
typedef struct cogdl_b200_hub_plan {
  int32_t chunk_edges;
  int32_t n_hub_rows;
  int32_t n_chunks;
  int32_t n_empty_rows;      /* rows of degree 0 (the row-stream kernels zero-fill them) */
  const int32_t *hub_rows;
  const int32_t *chunks;
  int32_t *counters;
  void *partials;
  int64_t partials_bytes;
  /* Row-stream segments (optional; segs == NULL => one warp per row).  A segment is a run of
   * consecutive NON-hub rows [row_begin, row_end) of roughly seg_cost rows+edges; its edges are
   * contiguous in colind, so one warp streams them in coalesced 32-edge slabs with always-full
   * gather batches and flushes its accumulator at row ends.  edge_row[p] = row owning edge p
   * (the COO row array) lets the kernel find row ends with one ballot per slab. */
  int32_t seg_cost;
  int32_t n_segs;
  const int32_t *segs;     /* [2*n_segs] (row_begin, row_end), any order */
  const int32_t *edge_row; /* [nnz] */
  /* Optional: HOST array of the hub rows' degrees, in hub_rows order, sorted DESCENDING (the caller
   * sorts hub_rows accordingly).  Lets row-tiered ops (edge softmax, GAT attention) launch exactly
   * as many blocks / clusters as there are rows in a tier.  NULL => such ops treat every hub row
   * with the per-warp tier. */
  const int32_t *hub_degrees_host;
} cogdl_b200_hub_plan_t;

/* Layout self-check for bindings that mirror the struct (ctypes, cgo, JNI): writes sizeof(cogdl_b200_hub_plan_t)
 * to out[0] and the byte offset of each field, in declaration order, to out[1..]; returns the number of values
 * written (at most n). */
COGDL_B200_API int cogdl_b200_hub_plan_layout(int64_t *out, int n);

/* Pass 1: counts_dev[0..3] = #rows with degree > chunk_edges, #chunks, #empty rows, #segments
 * (for seg_cost; pass seg_cost <= 0 to skip segments).  counts_dev: 4-int device buffer. */
COGDL_B200_API int cogdl_b200_hub_plan_count(const int32_t *rowptr, int64_t n_rows, int32_t chunk_edges,
                              int32_t seg_cost, int32_t *counts_dev, cogdl_b200_stream_t stream);
/* Pass 2: fills hub_rows[counts[0]], chunks[2*counts[1]] and segs[2*counts[3]] (caller-allocated
 * from pass 1's counts; segs may be NULL with seg_cost <= 0); counts_dev is reused as allocator. */
COGDL_B200_API int cogdl_b200_hub_plan_fill(const int32_t *rowptr, int64_t n_rows, int32_t chunk_edges,
                             int32_t seg_cost, int32_t *counts_dev, int32_t *hub_rows, int32_t *chunks,
                             int32_t *segs, cogdl_b200_stream_t stream);
/* edge_row[p] = row owning CSR position p (CSR -> COO row expansion; reference keeps the same
 * array as Adjacency.row, cogdl/data/data.py:136). */
COGDL_B200_API int cogdl_b200_edge_rows(const int32_t *rowptr, int64_t n_rows, int64_t nnz, int32_t *edge_row,
                         cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * CSR SpMM   Y[i,:] = sum_{p in row i} val[p] * X[colind[p],:]        (val == NULL => 1)
 * Replaces  spmm.csr_spmm(rowptr, colind, val, B)          cogdl/operators/spmm/spmm.cpp:22-45
 *           spmm.csr_spmm_no_edge_value(rowptr, colind, B) cogdl/operators/spmm/spmm.cpp:47-70
 *           (kernels spmm_test{0,1,2}, topo*SPMMKernel     .../spmm/spmm_kernel.cu:7-512)
 *           spmm_cpu.csr_spmm_cpu                          .../spmm/spmm_cpu.cpp:39-58 (semantics)
 * X is [n_src, F], Y is [n_rows, F]; colind values index rows of X.  Rows not split by a hub
 * plan are accumulated in CSR order with separate fp32 multiply and add, i.e. bit-identical
 * to the reference CPU SpMM (spmm_cpu.cpp:24-36).
 * Every SpMM entry below (fp32, fp16, residual, label propagation, device coefficient, accumulating,
 * two-source and peer forms) needs cogdl_b200_spmm_scratch_bytes(plan->n_chunks, F) bytes of plan->partials.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_spmm_scratch_bytes(int64_t n_chunks, int64_t F);
COGDL_B200_API int cogdl_b200_spmm_csr_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                            const float *X, float *Y, int64_t n_rows, int64_t F,
                            const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* Same, with X of x_rows rows and the column-panel count: when X is larger than the L2, the kernel makes one
 * pass over the graph per column panel of X (panel-major) so that the panel being gathered stays L2-resident;
 * the output is bit-identical whatever the panel count.  panels = 0 picks it from x_rows * F * 4 against the
 * device's L2 size (1 unless the plan has segments, F % 32 == 0 and the buffers are 16-byte aligned);
 * panels > 1 forces it (F / panels must be 32, 64 or 128, panels <= COGDL_B200_MAX_PANELS).
 * cogdl_b200_spmm_csr_f32 is this call with x_rows = n_rows and panels = 0. */
COGDL_B200_API int cogdl_b200_spmm_csr_f32_ex(const int32_t *rowptr, const int32_t *colind, const float *val,
                               const float *X, int64_t x_rows, float *Y, int64_t n_rows, int64_t F,
                               int32_t panels, const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* SpMM with a residual epilogue: the propagation step of GCNII / APPNP, `a * (r * (A @ X)) + b * Z`, in one launch.
 *   Y[i,:] = fl( fl(a * fl(r[i] * (A @ X)[i,:])) + fl(b * Z[i,:]) )
 * A @ X is cogdl_b200_spmm_csr_f32_ex's sum (same kernels, same accumulation order, same x_rows / panels / plan
 * rules, plan scratch sized as for it); each epilogue step is one fp32 multiply or add, so Y is bit-identical to the
 * SpMM followed by those operations one at a time.  row_scale ([n_rows], may be NULL: r = 1, no multiply) is the
 * in-degree normalisation applied after the SpMM; Z ([n_rows, F], may be NULL: no addition).  An empty row is the
 * epilogue of a zero sum.  x_rows must be the number of rows of X (every colind value is below it).  Y must not
 * overlap X (x_rows * F floats), Z or row_scale (COGDL_B200_EINVAL): they are still being read, through the read-only
 * cache, while finished rows of Y are written.  Z, when 16-byte aligned like X and Y, is read as float4. */
COGDL_B200_API int cogdl_b200_spmm_residual_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                               const float *X, int64_t x_rows, const float *Z, float a, float b,
                               const float *row_scale, float *Y, int64_t n_rows, int64_t F, int32_t panels,
                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* One label-propagation step of Correct & Smooth (outcome_correlation) in one launch: the residual epilogue of
 * cogdl_b200_spmm_residual_f32 followed by the post step.
 *   Y[i,:] = pin[i] ? Z[i,:] : clamp( fl( fl(a * fl(r[i] * (A @ X)[i,:])) + fl(b * Z[i,:]) ), lo, hi )
 * The clamp (has_clamp != 0) is torch.clamp's CUDA expression: a NaN passes, otherwise fminf(fmaxf(v, lo), hi).
 * pin ([n_rows] bytes, may be NULL) marks the rows reset to Z (a non-zero byte; needs Z), which are stored as Z's row
 * bit for bit.  Everything else -- sums, x_rows, panels, plan scratch, the alignment rules and the overlap checks
 * (COGDL_B200_EINVAL) -- is as for cogdl_b200_spmm_residual_f32. */
COGDL_B200_API int cogdl_b200_label_prop_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                               const float *X, int64_t x_rows, const float *Z, float a, float b,
                               const float *row_scale, const uint8_t *pin, int32_t has_clamp, float lo, float hi,
                               float *Y, int64_t n_rows, int64_t F, int32_t panels,
                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* The residual epilogue of cogdl_b200_spmm_residual_f32 with b read on the device: GIN's `(1 + eps) * x + A @ x`, with
 * a = 1 and b_dev pointing at fl(1 + eps), and its feature gradient over the adjoint.
 *   Y[i,:] = fl( fl(a * fl(r[i] * (A @ X)[i,:])) + fl((*b_dev) * Z[i,:]) )
 * b_dev is one fp32 value in device memory, read by the kernel (no host synchronisation); it is needed iff Z is given
 * and must not overlap Y.  Everything else -- sums, rounding, x_rows, panels, plan scratch, the alignment rules and the
 * overlap checks (COGDL_B200_EINVAL) -- is as for cogdl_b200_spmm_residual_f32. */
COGDL_B200_API int cogdl_b200_spmm_residual_dcoef_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                               const float *X, int64_t x_rows, const float *Z, float a, const float *b_dev,
                               const float *row_scale, float *Y, int64_t n_rows, int64_t F, int32_t panels,
                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* One hop of GRAND's random propagation in one launch: the SpMM, the in_norm and the running hop sum.
 *   Xn[i,:]  = fl(r[i] * (A @ X)[i,:])                       stored unless last != 0 (Xn may then be NULL)
 *   ACC[i,:] = fl(ACC_in[i,:] + Xn[i,:]), times scale (one fp32 multiply) when last != 0
 * acc_in may be NULL (ACC is updated in place) or another [n_rows, F] buffer that does not overlap ACC.  For
 * `y.div_(order + 1.0)` pass scale = fl(1 / (order + 1)): on CUDA torch divides by a host scalar as a multiply by its
 * fp32 reciprocal.  ACC must not overlap X or row_scale; Xn must not overlap X, ACC, acc_in or row_scale
 * (COGDL_B200_EINVAL).  Sums, x_rows, panels, plan scratch and the alignment rules (ACC and acc_in with Y) are as for
 * cogdl_b200_spmm_residual_f32. */
COGDL_B200_API int cogdl_b200_spmm_accum_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                               const float *X, int64_t x_rows, const float *row_scale, const float *acc_in, float *acc,
                               int32_t last, float scale, float *Xn, int64_t n_rows, int64_t F, int32_t panels,
                               const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* fp16 storage (X, val, Y are IEEE half), fp32 accumulation (the reference accumulates in
 * half, spmm_kernel.cu:222-250,311-368,442-512 -- documented divergence). */
COGDL_B200_API int cogdl_b200_spmm_csr_f16(const int32_t *rowptr, const int32_t *colind, const void *val,
                            const void *X, void *Y, int64_t n_rows, int64_t F,
                            const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* Two-source variant used by the node-range partitioned (multi-GPU) SpMM: column c reads
 * X0[c] when c < n0, else X1[c - n0] (X1 = halo rows received from / mapped on peers).
 * New functionality, no reference counterpart (SURVEY 8e). */
COGDL_B200_API int cogdl_b200_spmm_csr_f32_2src(const int32_t *rowptr, const int32_t *colind, const float *val,
                                 const float *X0, int64_t n0, const float *X1, float *Y,
                                 int64_t n_rows, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                 cogdl_b200_stream_t stream);

/* Peer form of the partitioned SpMM: the gather over remote feature rows is fused into the kernel.
 * A column c < n_local reads X_local[c]; a column c >= n_local encodes r = c - n_local with
 * owner = r >> owner_shift and row = r & ((1 << owner_shift) - 1), and is read DIRECTLY from
 * peer_ptrs[owner] -- that rank's feature shard mapped into this process (symmetric memory /
 * CUDA IPC), i.e. ld.global over NVLink 5 / NVSwitch inside the SpMM kernel: no pack kernel, no
 * all-to-all, no halo buffer.  peer_ptrs is a HOST array of n_peers (<= 8) device pointers.
 * Needs a hub plan with segments (row-stream kernel), F % 4 == 0, F <= 512.  The caller orders
 * the peers' writes to their shards before this call (barrier) -- see cogdl_b200/dist.py. */
COGDL_B200_API int cogdl_b200_spmm_csr_f32_peers(const int32_t *rowptr, const int32_t *colind, const float *val,
                                  const float *X_local, int64_t n_local, const float *const *peer_ptrs,
                                  int32_t n_peers, int32_t owner_shift, float *Y, int64_t n_rows, int64_t F,
                                  const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * CSR SDDMM   out[p] = < D1[row(p),:], D2[colind[p],:] >
 * Replaces  sddmm.csr_sddmm(rowptr, colind, D1, D2)   cogdl/operators/spmm/sddmm.cpp:47-70
 *           (kernels sddmmCSR{2,1}Scale               .../spmm/sddmm_kernel.cu:249-417)
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int cogdl_b200_sddmm_csr_f32(const int32_t *rowptr, const int32_t *colind, const float *D1,
                             const float *D2, float *out, int64_t n_rows, int64_t F,
                             const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * CSR -> CSC with permutation (integer only).
 * Replaces  spmm.csr2csc(rowptr, colind, val)   cogdl/operators/spmm/spmm.cpp:72-90
 *           (cuSPARSE cusparseCsr2cscEx2        .../spmm/spmm_kernel.cu:514-532,596-613)
 *           mhtranspose.csr2csc                 .../spmm/mhTranspose.cu:51-111
 * perm[q] = CSR position of CSC entry q; stable (inside a column, ascending row).  Values
 * are moved with cogdl_b200_gather_rows_f32(perm, ...) -- exact for any nnz (the reference
 * round-trips edge ids through fp32, wrong beyond 2^24 edges, mhspmm.py:55-59).
 * `workspace` is caller-provided device scratch of at least
 * cogdl_b200_csr2csc_workspace_bytes(nnz, n_cols) bytes.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_csr2csc_workspace_bytes(int64_t nnz, int64_t n_cols);
COGDL_B200_API int cogdl_b200_csr2csc(const int32_t *rowptr, const int32_t *colind, int64_t n_rows,
                       int64_t n_cols, int64_t nnz, int32_t *colptr, int32_t *rowind,
                       int32_t *perm, void *workspace, int64_t workspace_bytes,
                       cogdl_b200_stream_t stream);

/* out[q,:] = in[perm[q],:] over [nnz, H] fp32.
 * Replaces  mhtranspose.mhtranspose(perm, att)   cogdl/operators/spmm/mhTranspose.cu:6-49 */
COGDL_B200_API int cogdl_b200_gather_rows_f32(const int32_t *perm, const float *in, float *out, int64_t nnz,
                               int64_t H, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Edge softmax over the edges of each destination row, per head; [nnz, H] fp32.
 * Replaces  edge_softmax.edge_softmax(rowptr, w)               cogdl/operators/edge_softmax/edge_softmax.cc:16-31
 *           edge_softmax.edge_softmax_backward(rowptr, y, g)   .../edge_softmax.cc:33-49
 *           (kernels                                           .../edge_softmax.cu:7-98)
 * fwd: out = exp(in - max_row) / sum_row exp(in - max_row).  bwd: gin = y * (g - sum_row y*g).
 * Degree-0 rows own no entries, so nothing is written for them.
 * ------------------------------------------------------------------------------------- */
/* The calls below need cogdl_b200_edge_softmax_scratch_bytes(plan->n_chunks, H) bytes of plan->partials. */
COGDL_B200_API int64_t cogdl_b200_edge_softmax_scratch_bytes(int64_t n_chunks, int64_t H);
COGDL_B200_API int cogdl_b200_edge_softmax_fwd_f32(const int32_t *rowptr, const float *in, float *out,
                                    int64_t n_rows, int64_t H,
                                    const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_edge_softmax_bwd_f32(const int32_t *rowptr, const float *y, const float *g,
                                    float *gin, int64_t n_rows, int64_t H,
                                    const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Multi-head SpMM   out[i,h,:] = sum_p att[P(p),h] * feat[colind[p],h,:],  P(p) = perm ? perm[p] : p
 * Replaces  mhspmm.mhspmm(rowptr, colind, att, feat)   cogdl/operators/spmm/multiheadSpmm.cpp:8-34
 *           (kernels mhspmmSimple / mhspmm_1           .../spmm/multiheadSpmm.cu:6-51)
 * feat/out are [n, H, F]; att is [nnz, H].  `perm` fuses the backward's mhtranspose
 * (mhspmm.py:60-61) into the CSC pass.  Accumulation order/rounding as for SpMM.
 * plan->partials: cogdl_b200_mhspmm_scratch_bytes(plan->n_chunks, H, F) bytes (also for _dropout_f32).
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_mhspmm_scratch_bytes(int64_t n_chunks, int64_t H, int64_t F);
COGDL_B200_API int cogdl_b200_mhspmm_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                          const float *att, const float *feat, float *out, int64_t n_rows,
                          int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan,
                          cogdl_b200_stream_t stream);

/* Multi-head SDDMM   out[p,h] = < grad[row(p),h,:], feat[colind[p],h,:] >
 * Replaces  mhsddmm.mhsddmm(rowptr, colind, grad, feat)   cogdl/operators/spmm/multiheadSddmm.cu:6-113 */
COGDL_B200_API int cogdl_b200_mhsddmm_f32(const int32_t *rowptr, const int32_t *colind, const float *grad,
                           const float *feat, float *out, int64_t n_rows, int64_t H, int64_t F,
                           const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * scatter_max (neighbour max + argmax) and its backward.
 * Replaces  scatter_max.scatter_max_fp(rowptr, colind, x) -> [out, max_id]   cogdl/operators/scatter_max/scatter_max.cc:6-22
 *           scatter_max.scatter_max_bp(grad, max_id)                          .../scatter_max.cc:24-38
 *           (kernels                                                          .../scatter_max.cu:5-42)
 * fwd: out[i,f] = max_p X[colind[p],f]; argmax[i,f] = colind of the first edge (CSR order)
 *      attaining it.  Fixed semantics (documented divergences from the reference bugs):
 *      the running max starts at -inf (reference: FLT_MIN, scatter_max.cu:16); degree-0 rows
 *      give out = 0, argmax = -1 (reference: uninitialised max_id).  Identical to the
 *      reference whenever every row has a neighbour value > FLT_MIN.
 * bwd: gx[argmax[i,f], f] += g[i,f]; gx [n_src, F] is zero-filled by the call (the reference
 *      forgets to, scatter_max.cu:70); argmax < 0 is skipped.
 * fwd plan->partials: cogdl_b200_scatter_max_scratch_bytes(plan->n_chunks, F) bytes.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_scatter_max_scratch_bytes(int64_t n_chunks, int64_t F);
COGDL_B200_API int cogdl_b200_scatter_max_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *X,
                                   float *out, int32_t *argmax, int64_t n_rows, int64_t F,
                                   const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_scatter_max_bwd_f32(const float *g, const int32_t *argmax, float *gx,
                                   int64_t n_rows, int64_t n_src, int64_t F,
                                   cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * SortPool readout: the per-graph top-k selection.
 * Replaces  the padding, sorting and cutting of SortPool.forward   cogdl/models/nn/sortpool.py:105-126
 * (rowptr, colind) is the membership CSR: row g lists graph g's nodes (in ascending node order), n_graphs rows.
 * key_bits [n_x_rows] holds each node's key as the bit pattern of an IEEE binary32 value (SortPool's last channel),
 * ordered with integer operations only: every NaN above +inf, -0 equal to +0.
 * For each graph, the r-th of its min(k, n_g) nodes with the largest key, in descending key order with ties to the
 * lower node index (a stable descending torch.sort), is written to idx[g, r]; idx is -1 for r >= n_g.  The same
 * selection is written as a CSR of n_graphs * k rows: row g * k + r holds that node, or nothing for r >= n_g
 * (sel_rowptr [n_graphs * k + 1], sel_colind [sum of min(k, n_g)]), so cogdl_b200_spmm_csr_f32_ex over it with unit
 * values gathers the pooled rows and cogdl_b200_scatter_max_bwd_f32 with idx as the argmax scatters their gradient.
 * sel_off [n_graphs] must hold the exclusive prefix sum of min(k, n_g).  idx [n_graphs, k] int32.
 * 1 <= k <= cogdl_b200_sort_pool_max_k() (= COGDL_B200_SORT_POOL_MAX_K), else COGDL_B200_EINVAL before any launch.
 * ------------------------------------------------------------------------------------- */
#define COGDL_B200_SORT_POOL_MAX_K 1024
COGDL_B200_API int64_t cogdl_b200_sort_pool_max_k(void);
COGDL_B200_API int cogdl_b200_sort_pool_select(const int32_t *rowptr, const int32_t *colind, const uint32_t *key_bits,
                                int64_t n_x_rows, int64_t n_graphs, int64_t k, const int32_t *sel_off,
                                int32_t *idx, int32_t *sel_rowptr, int32_t *sel_colind,
                                cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * "Next" rows (SURVEY 8f).
 *
 * GAT forward: e = leakyrelu(h_l[i,h] + h_r[col,h]); a = softmax_row(e); out = sum a*feat.
 * The logits are formed and soft-maxed in registers (no [nnz,H] gather / add / activation
 * temporaries); the normalised attention is written once to att_out ([nnz,H], required: it is the
 * saved tensor of the backward and the operand of the row-stream multi-head SpMM that follows).
 * Replaces the unfused chain cogdl/layers/gat_layer.py:73-77 and the stale dgNN binding
 * cogdl/operators/fused_gat.py:17-19.
 * plan->partials: cogdl_b200_gat_fwd_scratch_bytes(plan->n_chunks, H, F) bytes (also for _dropout_f32).
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_gat_fwd_scratch_bytes(int64_t n_chunks, int64_t H, int64_t F);
COGDL_B200_API int cogdl_b200_gat_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *h_l,
                           const float *h_r, const float *feat, float negative_slope, float *out,
                           float *att_out, int64_t n_rows, int64_t H, int64_t F,
                           const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* GAT attention backward (SURVEY 8f-1; autograd of cogdl/layers/gat_layer.py:73-74, precedent
 * third_party/dgNN/dgNN/src/fused_gatconv/fused_gatconv_kernel.cu:636-790): softmax backward, LeakyReLU'
 * and the row sums in ONE pass over the edge-aligned tensors --
 *   d_edge[p,h] = att*(d_att - sum_row att*d_att) * leakyrelu'(h_l[row,h] + h_r[col,h])   [nnz,H]
 *   g_row[i,h]  = sum_{p in row i} d_edge[p,h]                                            [n_rows,H]
 * d_att is the multi-head SDDMM of (d out, feat).  g_col = cogdl_b200_edge_colsum_f32 over the transpose.
 * plan->partials: cogdl_b200_edge_softmax_scratch_bytes(plan->n_chunks, H) bytes (also for _dropout_f32). */
COGDL_B200_API int cogdl_b200_gat_attn_bwd_f32(const int32_t *rowptr, const int32_t *colind, const float *att,
                                const float *d_att, const float *h_l, const float *h_r, float negative_slope,
                                float *d_edge, float *g_row, int64_t n_rows, int64_t H,
                                const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
/* out[j,h] = sum_{q in column j of the transpose} e[perm[q], h]: column sums of an edge-aligned [nnz,H]
 * tensor through the cached CSC (colptr, perm).  Deterministic (no atomics; hub columns via the plan's chunks).
 * plan is the transpose's; its partials need cogdl_b200_edge_colsum_scratch_bytes(plan->n_chunks, H) bytes. */
COGDL_B200_API int64_t cogdl_b200_edge_colsum_scratch_bytes(int64_t n_chunks, int64_t H);
COGDL_B200_API int cogdl_b200_edge_colsum_f32(const int32_t *colptr, const int32_t *perm, const float *e, float *out,
                               int64_t n_cols, int64_t H, const cogdl_b200_hub_plan_t *plan,
                               cogdl_b200_stream_t stream);

/* GAT with attention dropout (the nn.Dropout between edge_softmax and mh_spmm in cogdl/layers/gat_layer.py:73-77).
 * Mask: (CSR edge position p, head h) is KEPT iff cogdl_b200_sample_draw(seed, p, h) >= drop_below, with
 * drop_below = floor(p_drop * 2^64) (0 keeps everything); a kept attention is multiplied by scale = 1 / (1 - p_drop)
 * (finite and > 0, else COGDL_B200_EINVAL).  p_drop = 1 has no kernel.
 * att_out receives the softmax with the SIGN BIT SET on the dropped entries (-a; the softmax is >= 0, and a dropped
 * softmax that underflowed to 0 is -0.0): one [nnz,H] tensor carries both the attention and the mask, and the
 * backward needs no seed.  The other arguments are those of cogdl_b200_gat_fwd_f32; with drop_below = 0 and
 * scale = 1 the results are bit-identical to it. */
COGDL_B200_API int cogdl_b200_gat_fwd_dropout_f32(const int32_t *rowptr, const int32_t *colind, const float *h_l,
                                   const float *h_r, const float *feat, float negative_slope, uint64_t seed,
                                   uint64_t drop_below, float scale, float *out, float *att_out, int64_t n_rows,
                                   int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
/* cogdl_b200_mhspmm_f32 over such a signed attention: an entry with the sign bit set counts as 0, the others as
 * att * scale.  With perm (the cached transpose) it is d feat of the dropout GAT. */
COGDL_B200_API int cogdl_b200_mhspmm_dropout_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                                  const float *att, const float *feat, float scale, float *out, int64_t n_rows,
                                  int64_t H, int64_t F, const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
/* cogdl_b200_gat_attn_bwd_f32 over such a signed attention; d_att = mhsddmm(d out, feat) is the gradient of the
 * dropped, scaled attention: the softmax backward runs on |att| with d_att * scale on the kept entries, 0 on the
 * dropped ones. */
COGDL_B200_API int cogdl_b200_gat_attn_bwd_dropout_f32(const int32_t *rowptr, const int32_t *colind, const float *att,
                                        const float *d_att, const float *h_l, const float *h_r, float negative_slope,
                                        float scale, float *d_edge, float *g_row, int64_t n_rows, int64_t H,
                                        const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Fused GCN layer (SURVEY 8f-3): OUT = act( (A.X).W^T + (A.1) b^T ), A = (rowptr, colind, val).
 * Equal to the reference layer  act( A.(X.W^T + 1 b^T) )  (cogdl/layers/gcn_layer.py:51-64, bias inside the
 * aggregation) up to fp32 rounding; the products are re-associated so the gather runs on the raw features
 * and the dense transform runs on the aggregated 128-row tile while it is on chip: bf16x3-split operands
 * (24 mantissa bits, six products), wgmma into registers, fp32 accumulate -- error vs fp64 ~1e-7 of the row
 * scale.  X [n_src,K], W [Fout,K] (torch.nn.Linear.weight layout), bias [Fout] or NULL, out [n_rows,Fout].
 * Needs K == 128, Fout <= 128 (cogdl_b200_gcn_fused_supported), a hub plan with edge_row, 16-byte aligned
 * X / W / out.  hub_agg: scratch [n_rows, K] fp32, required iff the plan has hub rows (only those rows are
 * written); plan->partials: cogdl_b200_gcn_fused_scratch_bytes(n_chunks, K) bytes.  rowsum: optional [n_rows]
 * = A.1 (sum of each row's edge values), worth caching when the edge weights are fixed (GCN); NULL =>
 * the kernel sums the weights itself (one warp per hub row: slow on 10^4-edge hubs).
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int cogdl_b200_gcn_fused_supported(int64_t K, int64_t Fout);
COGDL_B200_API int64_t cogdl_b200_gcn_fused_scratch_bytes(int64_t n_chunks, int64_t K);
COGDL_B200_API int cogdl_b200_gcn_fused_f32(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X,
                             const float *W, const float *bias, const float *rowsum, float *out, float *hub_agg, int64_t n_rows,
                             int64_t K, int64_t Fout, int32_t relu, const cogdl_b200_hub_plan_t *plan,
                             cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Fused GraphSAGE layer: OUT = act( S + agg(X).W_neigh^T ), the reference's  fc(cat[x, agg])
 * (cogdl/layers/sage_layer.py:69-87) with fc.weight = [W_self | W_neigh] and S = X[:n_rows].W_self^T + b
 * computed beforehand by the caller (the self half does not fit on chip beside the operand tiles).
 * The aggregation runs in the fused GCN kernel and the aggregated tile is never written to global memory:
 *   aggr == COGDL_B200_AGGR_SUM: agg = row_scale (.) (A.X), A = (rowptr, colind, val), val NULL = ones,
 *                                row_scale [n_rows] or NULL (graph.in_norm of a CSR-only graph; mean = sum
 *                                with row-normalised val or with row_scale = 1/deg).  Bit-identical to
 *                                row_scale * cogdl_b200_spmm_csr_f32(...).
 *   aggr == COGDL_B200_AGGR_MAX: agg = the values of cogdl_b200_scatter_max_fwd_f32 (strict `<` from -inf,
 *                                degree-0 rows 0), bit for bit; no argmax is produced.  val and row_scale
 *                                must be NULL.
 * The dense product is the bf16x3 wgmma of cogdl_b200_gcn_fused_f32 (~1e-7 of the row scale vs fp64).
 * X [n_src,K], W_neigh [Fout,K] contiguous, S and out [n_rows,Fout]; constraints as cogdl_b200_gcn_fused_f32
 * (cogdl_b200_gcn_fused_supported, hub plan with edge_row, 16-byte aligned X / W_neigh / S / out).
 * hub_agg: scratch [n_rows, K] fp32, required iff the plan has hub rows.  plan->partials:
 * cogdl_b200_sage_fused_scratch_bytes(n_chunks, K, aggr) bytes.
 * ------------------------------------------------------------------------------------- */
#define COGDL_B200_AGGR_SUM 0
#define COGDL_B200_AGGR_MAX 1
COGDL_B200_API int64_t cogdl_b200_sage_fused_scratch_bytes(int64_t n_chunks, int64_t K, int32_t aggr);
COGDL_B200_API int cogdl_b200_sage_fused_f32(const int32_t *rowptr, const int32_t *colind, const float *val,
                              const float *row_scale, const float *X, const float *W_neigh, const float *S, float *out,
                              float *hub_agg, int64_t n_rows, int64_t K, int64_t Fout, int32_t aggr, int32_t relu,
                              const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * GENConv softmax aggregation (DeeperGCN / RevGCN; cogdl/layers/deepergcn_layer.py:64-93) without per-edge
 * feature tensors.  Per row i, channel f, over the CSR edges e = (i, c_e):
 *   m_e = relu(X[c_e,f] + edge_term[e,f]) + eps        (edge_term: [nnz, F] in CSR order, or NULL)
 *   out[i,f] = sum_e w_e m_e,  w_e = softmax_e(beta m_e)       degree-0 rows: out = 0
 * beta is a DEVICE pointer to one float (a trainable parameter needs no host read; beta = 0 is the mean).
 * X is [n_cols, F], out / lse2 / Q are [n_rows, F].  Optional outputs for the backward:
 *   lse2[i,f] = log2 sum_e 2^(beta log2(e) m_e)   (base-2 log-sum-exp of the logits)
 *   Q[i,f]    = sum_e w_e m_e^2                   (d out / d beta = Q - out^2)
 * Any F >= 1; 16-byte vectors when F % 4 == 0 and every buffer is 16-byte aligned.  Hub rows are cut into the
 * plan's chunks and merged in chunk order (no float atomics: bit-reproducible).  plan->partials needs
 * cogdl_b200_softmax_aggr_scratch_bytes(n_chunks, F) bytes.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_softmax_aggr_scratch_bytes(int64_t n_chunks, int64_t F);
COGDL_B200_API int cogdl_b200_softmax_aggr_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *X,
                                    const float *edge_term, const float *beta, float eps, float *out, float *lse2,
                                    float *Q, int64_t n_rows, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                    cogdl_b200_stream_t stream);
/* Backward over the transpose (colptr, rowind, perm of cogdl_b200_csr2csc; n_cols columns), given G = dL/dout and
 * the forward's out and lse2:
 *   dpre_e = G[i] w_e (1 + beta (m_e - out[i])) [X[j] + edge_term[e] > 0]
 *   dX[j] = sum_{e: c_e = j} dpre_e  (transpose order; hub columns through `plan`, the TRANSPOSE's plan, whose
 *           partials need cogdl_b200_softmax_aggr_bwd_scratch_bytes(n_chunks, F) bytes)
 *   d_edge_term[e] = dpre_e  (optional, needs edge_term)
 * perm is needed only with an edge term.  d beta = sum G (Q - out^2) is left to the caller. */
COGDL_B200_API int64_t cogdl_b200_softmax_aggr_bwd_scratch_bytes(int64_t n_chunks, int64_t F);
COGDL_B200_API int cogdl_b200_softmax_aggr_bwd_f32(const int32_t *colptr, const int32_t *rowind, const int32_t *perm,
                                    const float *X, const float *edge_term, const float *beta, float eps,
                                    const float *G, const float *out, const float *lse2, float *dX,
                                    float *d_edge_term, int64_t n_cols, int64_t F, const cogdl_b200_hub_plan_t *plan,
                                    cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * GENConv softmax aggregation with a linear edge encoder (EdgeEncoder, cogdl/layers/deepergcn_layer.py:168-174:
 * nn.Linear(D, F, bias=False)), the edge term formed in registers instead of read from an [nnz, F] tensor:
 *   edge_term[e,f] = sum_{d=0..D-1} attr[e,d] W[f,d]   (one fmaf chain, d ascending)
 * and otherwise the operation of cogdl_b200_softmax_aggr_fwd_f32 / _bwd_f32, with the same work items, hub plan,
 * chunk-order merge and lse2 / Q outputs.  attr is [nnz, D] fp32 in CSR order, W is [F, D] fp32 (nn.Linear layout),
 * 1 <= D <= 16 (wider D is rejected).  The forward's plan->partials needs cogdl_b200_softmax_aggr_scratch_bytes(n_chunks,
 * F) bytes.  When F is a multiple of 4, 16-byte vectors if X, out, lse2, Q (and G, dX, the partials) are aligned.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int cogdl_b200_genconv_edge_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *X,
                                                   const float *attr, const float *W, int64_t D, const float *beta,
                                                   float eps, float *out, float *lse2, float *Q, int64_t n_rows,
                                                   int64_t F, const cogdl_b200_hub_plan_t *plan,
                                                   cogdl_b200_stream_t stream);
/* Backward over the transpose (colptr, rowind, perm; n_cols columns; `plan` is the TRANSPOSE's plan, partials
 * cogdl_b200_genconv_edge_bwd_scratch_bytes(n_chunks, F, dX != NULL) bytes), given G = dL/dout and the forward's out
 * and lse2:
 *   dX[j]    = sum_{e: c_e = j} dpre_e             (as cogdl_b200_softmax_aggr_bwd_f32; NULL: not computed)
 *   dW[f,d]  = sum_e dpre_e[f] attr[e,d]           ([F, D]; NULL: not computed)
 * dW is summed without float atomics: per warp over a fixed, static assignment of work items, then per block in warp
 * order into dw_scratch, then over the blocks in block order, so it is bit-identical run to run on one device.
 * dw_scratch must hold cogdl_b200_genconv_edge_dw_scratch_bytes(F, D) bytes (a bound independent of nnz).  At least
 * one of dX, dW.  d beta = sum G (Q - out^2) is left to the caller. */
COGDL_B200_API int64_t cogdl_b200_genconv_edge_dw_scratch_bytes(int64_t F, int64_t D);
COGDL_B200_API int64_t cogdl_b200_genconv_edge_bwd_scratch_bytes(int64_t n_chunks, int64_t F, int32_t want_dx);
COGDL_B200_API int cogdl_b200_genconv_edge_bwd_f32(const int32_t *colptr, const int32_t *rowind, const int32_t *perm,
                                                   const float *X, const float *attr, const float *W, int64_t D,
                                                   const float *beta, float eps, const float *G, const float *out,
                                                   const float *lse2, float *dX, float *dW, float *dw_scratch,
                                                   int64_t dw_scratch_bytes, int64_t n_cols, int64_t F,
                                                   const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * DisenGCN neighbourhood routing, one step (cogdl/layers/disengcn_layer.py:40-91) without per-edge feature
 * tensors.  Rows of F = K*d floats are K channels of d (channel k = columns [k*d, (k+1)*d)).  c holds the
 * per-(node, channel) normalised features, q the current routing state ([n, F] each).  Per row i, channel k,
 * over the CSR edges e = (i, j):
 *   s_e = (q[i,k] . c[j,k]) / tau,  w_e = softmax over row i's edges of s_e,  u = sum_e w_e c[j,k] + c[i,k]
 *   out[i,k] = u / |u|           (degree-0 rows: u = c[i,k]; |u| = 0 gives NaN, as the reference)
 * Optional training outputs, [n, K], both or neither:
 *   lse2[i,k] = log2 sum_e 2^(s_e log2 e)   (base-2 log-sum-exp of the logits)      r[i,k] = |u|
 * The structure must be square (n_rows == n_cols); F % K == 0; d = F/K a power of two from 1 to 32; tau > 0.
 * 16-byte vectors when d % 4 == 0 and every feature buffer is 16-byte aligned.  Hub rows are cut into the plan's
 * chunks and merged in chunk order (no float atomics: bit-reproducible).  plan->partials needs
 * cogdl_b200_disen_route_scratch_bytes(n_chunks, F, K) bytes.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_disen_route_scratch_bytes(int64_t n_chunks, int64_t F, int64_t K);
COGDL_B200_API int cogdl_b200_disen_route_fwd_f32(const int32_t *rowptr, const int32_t *colind, const float *q,
                                   const float *c, float *out, float *lse2, float *r, int64_t n_rows,
                                   int64_t n_cols, int64_t F, int64_t K, float tau,
                                   const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
/* Backward of one step, given G = dL/dout and the forward's out, lse2 and r.  Two kernels:
 *   row kernel (CSR rowptr/colind, its plan `plan`): g_u = (G - out (out . G)) / r into the caller's scratch
 *     g_u [n, F]; with t_e = g_u[i] . c[j] and D[i,k] = sum_e w_e t_e (into the scratch D [n, K]),
 *     dq[i] = sum_e w_e (t_e - D[i]) c[j] / tau
 *   column kernel (transpose colptr/rowind of cogdl_b200_csr2csc, ITS plan `plan_t`):
 *     dc[j] = g_u[j] + sum_{e=(i,j)} [w_e g_u[i] + w_e (t_e - D[i]) q[i] / tau]
 * w_e is recomputed from lse2.  plan and plan_t each need cogdl_b200_disen_route_scratch_bytes(n_chunks, F, K) bytes of
 * partials, with that plan's n_chunks; hub rows / columns are merged in chunk order.  dq and dc are overwritten. */
COGDL_B200_API int cogdl_b200_disen_route_bwd_f32(const int32_t *rowptr, const int32_t *colind,
                                   const cogdl_b200_hub_plan_t *plan, const int32_t *colptr,
                                   const int32_t *rowind, const cogdl_b200_hub_plan_t *plan_t, const float *q,
                                   const float *c, const float *G, const float *out, const float *lse2,
                                   const float *r, float *g_u, float *D, float *dq, float *dc, int64_t n_rows,
                                   int64_t n_cols, int64_t F, int64_t K, float tau, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * CompGCN composition aggregation (cogdl/models/nn/compgcn.py:124-140) without per-edge feature tensors.
 * Per row i of the CSR (rowptr, colind) with per-slot second index idx2 and weight w:
 *   Y[i,:] = sum_{q in row i} w[q] * phi(A[colind[q],:], B[idx2[q],:])
 *   op COGDL_B200_COMP_MULT: phi = a * b;  COGDL_B200_COMP_SUB: phi = a - b;  COGDL_B200_COMP_COPY: phi = a (idx2
 *   and B unused, may be NULL).
 * A is [a_rows, F], B [b_rows, F], Y [n_rows, F], all fp32 row-major; colind < a_rows and idx2 < b_rows are the
 * caller's to guarantee.  Degree-0 rows give zeros.  Needs a hub plan (chunk_edges > 0) with row-stream
 * segments; plan->partials needs cogdl_b200_comp_aggr_scratch_bytes(n_chunks, F) bytes.  Hub rows are merged in
 * chunk order (no float atomics: bit-reproducible).  16-byte vectors when F % 4 == 0 and A, B, Y and the partials
 * are 16-byte aligned.  Rejects an unknown op, F <= 0 and a plan whose row counts do not match n_rows.
 * ------------------------------------------------------------------------------------- */
#define COGDL_B200_COMP_MULT 0
#define COGDL_B200_COMP_SUB 1
#define COGDL_B200_COMP_COPY 2
COGDL_B200_API int64_t cogdl_b200_comp_aggr_scratch_bytes(int64_t n_chunks, int64_t F);
COGDL_B200_API int cogdl_b200_comp_aggr_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *idx2,
                                            const float *w, const float *A, int64_t a_rows, const float *B,
                                            int64_t b_rows, float *Y, int64_t n_rows, int64_t F, int32_t op,
                                            const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * R-GCN relational aggregation under a basis decomposition (cogdl/layers/rgcn_layer.py:118-150), without a
 * per-relation tensor.  Per row i of the CSR (rowptr, colind) with per-slot edge type etype and weight w, and a
 * coefficient table coef [T, B] (etype < T is the caller's to guarantee):
 *   cogdl_b200_rgcn_aggr_f32:      Y[i,b,:] = sum_{q in row i} fl(w[q] * coef[etype[q], b]) * X[colind[q], :]
 *                                  (per_basis != 0: X is [*, B, F] and basis b gathers X[colind[q], b, :])
 *   cogdl_b200_rgcn_edge_dot_f32:  P[q, b]  = fl(w[q] * <G[i, b, :], X[colind[q], :]>) for every slot q of row i
 * X [*, F] (or [*, B, F]), Y and G [n_rows, B, F], P [nnz, B], all fp32 row-major.  Degree-0 rows give zeros.  Y[:, b, :]
 * is accumulated in CSR order with a separate multiply and add and hub rows are merged in chunk order, so it is
 * bit-identical to cogdl_b200_spmm_csr_f32_ex with values fl(w * coef[etype, b]) on the same plan; both entries are
 * reproducible run to run (no float atomics).  Needs a hub plan (chunk_edges > 0) with row-stream segments; for the
 * aggregation plan->partials needs cogdl_b200_rgcn_aggr_scratch_bytes(n_chunks, B, F) bytes.  16-byte vectors when
 * F % 4 == 0 and the feature buffers (and the partials) are 16-byte aligned.  Rejects F <= 0, B outside [1, 4096] and a
 * plan whose row counts do not match n_rows.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_rgcn_aggr_scratch_bytes(int64_t n_chunks, int64_t B, int64_t F);
COGDL_B200_API int cogdl_b200_rgcn_aggr_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *etype,
                                            const float *w, const float *coef, int64_t B, const float *X,
                                            int32_t per_basis, float *Y, int64_t n_rows, int64_t F,
                                            const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_rgcn_edge_dot_f32(const int32_t *rowptr, const int32_t *colind, const float *w,
                                                const float *G, const float *X, float *P, int64_t n_rows, int64_t B,
                                                int64_t F, const cogdl_b200_hub_plan_t *plan,
                                                cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Simple-HGN attention (myGATConv, CogDL examples/simple_hgn/conv.py): the GAT attention stage with an edge-type
 * term and the residual attention blend.  Per CSR edge p = (i, j) of type t = etype[p] (int32, in [0, T): the
 * caller's to guarantee) and head h, with h_e [T, H]:
 *   a[p,h]        = softmax over row i of leakyrelu(h_l[i,h] + h_r[j,h] + h_e[t,h])
 *   att_out[p,h]  = a with the sign bit set when dropped (optional: NULL when no gradient is needed)
 *   mix_out[p,h]  = (1 - alpha) * (dropped ? 0 : a * scale) + alpha * res_attn[p,h]   (res_attn NULL: no blend)
 * Dropout, seed and keep rule are those of cogdl_b200_gat_fwd_dropout_f32 (drop_below = 0 keeps everything; scale
 * finite and > 0).  mix_out is what the layer aggregates (cogdl_b200_mhspmm_f32) and returns.
 * cogdl_b200_hgn_attn_bwd_f32, given att (att_out of the forward) and d_mix = mhsddmm(d out, feat), writes
 *   d_edge[p,h] = |a| * (g - sum_row |a| * g) * leakyrelu'(h_l[i,h] + h_r[j,h] + h_e[t,h])   [nnz, H]
 *   g_row[i,h]  = sum_{p in row i} d_edge[p,h]                                                [n_rows, H]
 * with g = (sign bit of att) ? 0 : d_mix * grad_scale, grad_scale = (1 - alpha) / (1 - p_drop).
 * T * H must be in [1, cogdl_b200_hgn_max_table()] (h_e is staged in shared memory), else COGDL_B200_EINVAL before
 * any launch.  Any H; plan->partials needs cogdl_b200_edge_softmax_scratch_bytes(plan->n_chunks, H) bytes.
 * cogdl_b200_last_kernel() names every launch (hgn_warp_kernel / hgn_generic_kernel / [hgn_stats_kernel +]
 * hgn_main_kernel).
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_hgn_max_table(void);
COGDL_B200_API int cogdl_b200_hgn_attn_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *etype,
                                           const float *h_l, const float *h_r, const float *h_e, int64_t T,
                                           float negative_slope, uint64_t seed, uint64_t drop_below, float scale,
                                           const float *res_attn, float alpha, float *att_out, float *mix_out,
                                           int64_t n_rows, int64_t H, const cogdl_b200_hub_plan_t *plan,
                                           cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_hgn_attn_bwd_f32(const int32_t *rowptr, const int32_t *colind, const int32_t *etype,
                                               const float *att, const float *d_mix, const float *h_l,
                                               const float *h_r, const float *h_e, int64_t T, float negative_slope,
                                               float grad_scale, float *d_edge, float *g_row, int64_t n_rows,
                                               int64_t H, const cogdl_b200_hub_plan_t *plan,
                                               cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Sparse x sparse product C = A.B, A [a_rows x a_cols] and B [b_rows x b_cols] int32 CSR with fp32 values, columns
 * ascending and unique inside every row (b_rows must equal a_cols).  C comes out as CSR with ascending, unique columns.
 * Replaces  torch_sparse.spspmm(indexA, valueA, indexB, valueB, m, k, n)   (cuSPARSE SpGEMM), imported at module level
 *           by cogdl/models/nn/gtn.py:7 (GTLayer.forward :82), cogdl/models/nn/srgcn.py:6 (nhop powers :79,153),
 *           cogdl/utils/srgcn_utils.py:7 (NodeAttention :36, PPR :133) and cogdl/models/nn/graph_unet.py:9 (:38).
 * The pattern is structural: (i, j) is in C when some product a_ik b_kj exists, even if the values sum to 0.
 * Every value is acc = fmaf(a_ik, b_kj, acc) from 0, in (A's CSR order, B's CSR order), without float atomics: rows
 * are never split, so C is bit-identical to that sequential loop and reproducible run to run.
 *   1. ..._count  : rowptrC[a_rows+1] and *nnz_c (host) = nnz(C).  Totals are int64; nnz(C) > INT32_MAX returns
 *                   EINVAL with nothing written to rowptrC.  Reads the total on the host (synchronises the stream).
 *   2. ..._fill   : colC / valC [nnz(C)], caller-allocated from step 1.
 * `scratch`: device memory of at least cogdl_b200_spgemm_scratch_bytes(a_rows, a_cols, b_cols) bytes, for both steps
 * (about 28 bytes per row of A plus 33 bytes per column of B; the per-column part, a bitmap and its prefix sums for each
 * of 132 concurrent rows, is written only when a row has more than 4096 possible columns).
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int64_t cogdl_b200_spgemm_scratch_bytes(int64_t a_rows, int64_t a_cols, int64_t b_cols);
COGDL_B200_API int cogdl_b200_spgemm_count(const int32_t *rowptrA, const int32_t *colA, int64_t a_rows, int64_t a_cols,
                                           const int32_t *rowptrB, const int32_t *colB, int64_t b_rows, int64_t b_cols,
                                           int32_t *rowptrC, int64_t *nnz_c, void *scratch, int64_t scratch_bytes,
                                           cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_spgemm_fill_f32(const int32_t *rowptrA, const int32_t *colA, const float *valA,
                                              int64_t a_rows, int64_t a_cols, const int32_t *rowptrB, const int32_t *colB,
                                              const float *valB, int64_t b_rows, int64_t b_cols, const int32_t *rowptrC,
                                              int32_t *colC, float *valC, void *scratch, int64_t scratch_bytes,
                                              cogdl_b200_stream_t stream);
/* Value gradients of C = A.B given dC [nnz(C)] (the backward of torch_sparse.spspmm's values; GTN's GTConv weights
 * train only through them):
 *   dA[p=(i,k)] = sum_{q in B_k} b_q dC[i, col_B(q)]                      (dA [nnz(A)], NULL = not wanted)
 *   dB[q=(k,j)] = sum_{p in column k of A} a_p dC[row(p), j]              (dB [nnz(B)], NULL = not wanted)
 * dB walks A's transpose: colptrAT / rowindAT / permAT of cogdl_b200_csr2csc (needed only with dB).  Each output is
 * written once by one warp (fixed-order lane sums): deterministic. */
COGDL_B200_API int cogdl_b200_spgemm_bwd_f32(const int32_t *rowptrA, const int32_t *colA, const float *valA,
                                             int64_t a_rows, int64_t a_cols, const int32_t *rowptrB, const int32_t *colB,
                                             const float *valB, int64_t b_rows, int64_t b_cols, const int32_t *rowptrC,
                                             const int32_t *colC, const float *dC, const int32_t *colptrAT,
                                             const int32_t *rowindAT, const int32_t *permAT, float *dA, float *dB,
                                             cogdl_b200_stream_t stream);

/* Device COO -> CSR (stable): row_ptr[num_nodes+1] and reindex[nnz] (CSR slot -> COO position),
 * int64 as cogdl.data.Graph stores them.
 * Replaces  sampler.coo2csr_cpu_index(row, col, num_nodes)   cogdl/operators/sample/sample.cpp:234-270
 * (single-thread CPU counting sort even for CUDA graphs, cogdl/utils/graph_utils.py:133-142). */
COGDL_B200_API int64_t cogdl_b200_coo2csr_workspace_bytes(int64_t nnz, int64_t num_nodes);
COGDL_B200_API int cogdl_b200_coo2csr_index(const int64_t *row, int64_t nnz, int64_t num_nodes, int64_t *row_ptr,
                             int64_t *reindex, void *workspace, int64_t workspace_bytes,
                             cogdl_b200_stream_t stream);

/* int64 -> int32 narrowing of CSR arrays (fails with EINVAL semantics left to the caller: values
 * must fit).  Replaces the per-call `.int()` casts of cogdl/utils/spmm_utils.py:106. */
COGDL_B200_API int cogdl_b200_narrow_i64_i32(const int64_t *in, int32_t *out, int64_t n, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Neighbour sampling and induced subgraphs on the device (SURVEY 8f-4).  int64 CSR in / int64 out, as
 * cogdl.data.Graph stores it (row_ptr, col).
 * Replaces  sampler.sample_adj(indptr, indices, node_idx, num_neighbors, replace)
 *             -> (out_indptr, out_indices, out_nodes, out_edges)   cogdl/operators/sample/sample.cpp:6-146
 *           sampler.subgraph(indptr, indices, node_idx)
 *             -> (out_indptr, out_indices, arange, out_edges)      cogdl/operators/sample/sample.cpp:148-188
 * (single-thread host loops called per mini-batch by Graph.sample_adj / csr_subgraph, data.py:792-874).
 *
 * Results are IDENTICAL to the reference's sequential loops for any emitted edge list: out_nodes =
 * batch nodes, then new source nodes in order of first appearance; out_indices = their positions.
 * Which edges are emitted: num_neighbors < 0 -> every edge of each batch row (CSR order);
 * replace != 0 -> num_neighbors draws with replacement per row (none for a degree-0 row; the
 * reference divides by zero there); else min(deg, num_neighbors) DISTINCT edges by Floyd's algorithm
 * in insertion order (the reference's variant draws `rand() % j` and is biased -- fixed, see
 * sampler.cu).  Every draw is cogdl_b200_sample_draw(seed, batch slot, draw index): a counter-based
 * generator, so batches are reproducible and bit-checkable (the reference uses unseeded libc rand()).
 *
 * Two phases because the output sizes are data dependent and the caller owns every buffer:
 *   1. ..._count : out_indptr[n_batch+1] (device).  Read out_indptr[n_batch] = n_edges on the host.
 *   2. ..._fill  : out_indices / out_edges [n_edges], out_nodes [capacity n_batch + n_edges],
 *                  *n_out_nodes_dev (device int64) = number of out_nodes entries written.
 * `assoc`: device int32[num_nodes] scratch, every entry COGDL_B200_SAMPLE_UNSEEN on entry; restored
 * before the fill returns (subgraph: marked by _count, restored by _fill -- always call both).
 * node_idx entries must be distinct.  n_batch + n_edges must fit int32.
 * `workspace`: >= cogdl_b200_sample_workspace_bytes(n_batch, n_edges) bytes (n_edges = 0 for _count).
 * ------------------------------------------------------------------------------------- */
#define COGDL_B200_SAMPLE_UNSEEN 0x7fffffff
COGDL_B200_API uint64_t cogdl_b200_sample_draw(uint64_t seed, int64_t slot, int64_t k);
COGDL_B200_API int64_t cogdl_b200_sample_workspace_bytes(int64_t n_batch, int64_t n_edges);
COGDL_B200_API int cogdl_b200_sample_adj_count(const int64_t *indptr, const int64_t *node_idx, int64_t n_batch,
                                int64_t num_neighbors, int32_t replace, int64_t *out_indptr, void *workspace,
                                int64_t workspace_bytes, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_sample_adj_fill(const int64_t *indptr, const int64_t *indices, const int64_t *node_idx,
                               int64_t n_batch, int64_t num_nodes, int64_t num_neighbors, int32_t replace,
                               uint64_t seed, const int64_t *out_indptr, int64_t n_edges, int32_t *assoc,
                               int64_t *out_indices, int64_t *out_edges, int64_t *out_nodes,
                               int64_t *n_out_nodes_dev, void *workspace, int64_t workspace_bytes,
                               cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_subgraph_count(const int64_t *indptr, const int64_t *indices, const int64_t *node_idx,
                              int64_t n_sub, int32_t *assoc, int64_t *out_indptr, void *workspace,
                              int64_t workspace_bytes, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_subgraph_fill(const int64_t *indptr, const int64_t *indices, const int64_t *node_idx,
                             int64_t n_sub, int32_t *assoc, const int64_t *out_indptr, int64_t *out_indices,
                             int64_t *out_edges, cogdl_b200_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Activation-compressed training (ActNN's activation quantization, third_party/actnn; actnn.cu has the rules).
 *
 * x: [N, D] fp32 row-major; D is zero-padded to Dp = ceil(D / group_size) * group_size, group_size 64 or 256,
 * G = Dp / group_size groups per row.
 * _minmax: mn, mx [N * G] fp32 = min / max of each padded group (the C of the bit allocation is built from them).
 * _pack: codes of every padded element; scale_bf16 / mn_bf16 [N * G] bf16.  Bit widths: bits = NULL and
 *   uniform_bits in {1, 2, 4, 8}, packed = N * Dp * uniform_bits / 8 bytes; or bits [N] int32 in 1..8 with
 *   row_offsets [N] int64 = exclusive prefix sum of bits * Dp / 8, packed = sum(bits) * Dp / 8 bytes.
 *   stochastic != 0 adds draw(seed, n * Dp + d, 0) noise (rng.cuh) before rounding; 0 rounds to nearest.
 * _unpack: out [N, D] fp32 = code / scale + mn, same width arguments as the pack.
 * Masks: uint32 [ceil(n / 32)] words, bit i % 32 of word i / 32 = element i.  The dropout keeps element i iff
 *   draw(seed, i, 0) >= drop_below (= floor(p * 2^64)) and scales it by 1 / (1 - p); p in [0, 1).
 * _bits: the reference greedy (calc_precision.cc, w = 1) on the device: bits [N] from initial_bits (1..8) down to at
 *   least 1 until sum(bits) <= target.  C [N] fp32 must be finite and >= 0 (else EINVAL; one 4-byte status word is
 *   read back, C is not).  N < 2^28; scratch >= cogdl_b200_actnn_bits_scratch_bytes(N) bytes of device memory.
 * ------------------------------------------------------------------------------------- */
COGDL_B200_API int cogdl_b200_actnn_minmax_f32(const float *x, int64_t N, int64_t D, int32_t group_size, float *mn,
                                float *mx, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_actnn_pack_f32(const float *x, int64_t N, int64_t D, int32_t group_size,
                              const int32_t *bits, int32_t uniform_bits, const int64_t *row_offsets,
                              int32_t stochastic, uint64_t seed, uint8_t *packed, void *scale_bf16, void *mn_bf16,
                              cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_actnn_unpack_f32(const uint8_t *packed, int64_t N, int64_t D, int32_t group_size,
                                const int32_t *bits, int32_t uniform_bits, const int64_t *row_offsets,
                                const void *scale_bf16, const void *mn_bf16, float *out, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_actnn_relu_fwd_f32(const float *x, int64_t n, float *y, uint32_t *mask,
                                  cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_actnn_relu_bwd_f32(const float *g, const uint32_t *mask, int64_t n, float *gx,
                                  cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_actnn_dropout_fwd_f32(const float *x, int64_t n, float p, uint64_t seed,
                                     uint64_t drop_below, float *y, uint32_t *mask, cogdl_b200_stream_t stream);
COGDL_B200_API int cogdl_b200_actnn_dropout_bwd_f32(const float *g, const uint32_t *mask, int64_t n, float p,
                                     float *gx, cogdl_b200_stream_t stream);
COGDL_B200_API int64_t cogdl_b200_actnn_bits_scratch_bytes(int64_t N);
COGDL_B200_API int cogdl_b200_actnn_bits(const float *C, int64_t N, int32_t initial_bits, int64_t target,
                          int32_t *bits, void *scratch, int64_t scratch_bytes, cogdl_b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* COGDL_B200_H_ */

// stream.cuh -- the row-stream gather kernel shared by the SpMM (with each of its store epilogues), the multi-head SpMM
// and the CompGCN composition aggregation (sm_90a).
//
// Work items, in grid order:
//   [0, n_chunks)                 hub chunks: <= chunk_edges edges of ONE hub row -> partial sum in
//                                 scratch, combined in chunk order by the last chunk to arrive;
//   [n_chunks, n_chunks+n_segs)   segments: runs of consecutive NON-hub rows (~seg_cost rows+edges).
// In multi-head mode every item exists once per 512-byte slice of the [H*F] row (adjacent warps).
// In panel mode (plain SpMM, X larger than the L2) every item exists once per column panel of X, panel-major:
// blockIdx.y = panel.  Blocks are dispatched roughly in linear block order (x fastest), so about one panel
// of X (F/S columns of every row) is live in the L2 at a time and each X line is fetched from DRAM ~once.
//
// One warp per item.  A segment's edges are contiguous in colind/val/edge_row, so the warp walks
// them in 32-edge slabs: one coalesced load each for colind, the value (or permutation) and the
// owning row; `row != row of the next edge` gives a 32-bit "row ends here" mask with one ballot.
// Gathers are issued U at a time and are always full batches except at the segment tail, whatever
// the row lengths (a row-per-warp kernel issues only `degree` gathers behind a rowptr -> colind -> X
// dependent chain).  Per output element the accumulation is strictly in CSR order with separate
// fp32 multiply and add => bit-identical to the reference CPU loop (spmm_cpu.cpp:24-36) for every
// row that is not a hub.  At a set mask bit the accumulator is stored to its row and cleared.
#pragma once
#include "common.cuh"

namespace cogdl_b200 {

// The operands of the plain SpMM's store epilogue (EPI below), a member of StreamParams and of SpmmParams (spmm.cuh).
struct SpmmEpilogue {
  // residual epilogue (spmm_residual.cu, EPI_RESID): every finished row i is written as
  // fl(fl(res_a * fl(row_scale[i] * acc)) + fl(res_b * Z[i])); row_scale and Z are optional ([n_rows], [n_rows, ldv]).
  const float *Z = nullptr;
  const float *row_scale = nullptr;
  float res_a = 1.f, res_b = 0.f;
  // label-propagation epilogue (label_prop.cu, EPI_LABELPROP): the residual epilogue's value, clamped to
  // [clamp_lo, clamp_hi] as torch.clamp does when has_clamp; a row i with pin[i] != 0 stores Z[i] instead.  pin
  // ([n_rows] bytes) is optional and needs Z.
  const unsigned char *pin = nullptr;
  int has_clamp = 0;
  float clamp_lo = 0.f, clamp_hi = 0.f;
  // residual epilogue with a device coefficient (gin.cu, EPI_RESID_DEV): the residual epilogue with res_b read from
  // *res_b_dev (one fp32 value in device memory) instead of res_b.
  const float *res_b_dev = nullptr;
  // accumulating epilogue (spmm_accum.cu, EPI_ACCUM): v = fl(row_scale[i] * acc) is stored to Y[i] unless acc_last,
  // and ACC[i] = fl(Z[i] + v), times acc_scale (fl) when acc_last.  Z is ACC's input: ACC itself (in place) or another
  // buffer of Y's layout; Y is ACC when acc_last (nothing else is written).
  float *acc = nullptr;
  int acc_last = 0;
  float acc_scale = 1.f;
};

struct StreamParams {
  const int *rowptr;
  const int *colind;
  const float *val;   // MODE 1: [nnz]; null => unweighted
  const float *att;   // MODE 2: [nnz, H]
  const int *perm;    // MODE 2, nullable: attention row of edge p is perm[p]
  const float *X0;
  const float *X1;    // second source (two-source form), rows >= n0
  int64_t n0;
  // peer form (node-range partition, fused NVLink gather): a column c >= n0 encodes
  // (owner << peer_shift | row inside the owner's shard) after subtracting n0; peers[owner] is that
  // rank's feature shard mapped into this process (symmetric memory / CUDA IPC).
  const float *peers[8];
  int n_peers;
  int peer_shift;
  float *Y;
  int ldv;            // dense row length in VecT units
  int H;              // MODE 2: heads
  int FVL;            // MODE 2: VecT units per head
  int S;              // MODE 2: 512-byte slices per row; panel mode: column panels of 32 VecT (1 otherwise)
  HubView hub;
  // composition modes (comp_aggr.cu): edge q also reads B[idx2[q]] ([*, ldv], like X0) and accumulates
  // val[q] * (X0[colind[q]] o B[idx2[q]]) with o = * (MODE_COMP_MULT) or - (MODE_COMP_SUB)
  const int *idx2;
  const float *B;
  // multi-head form with DROP: the attention carries an attention-dropout mask in its sign bit (edge_softmax.cu,
  // MODE 2); a kept entry is read as att * drop_scale, a dropped one as |att| * 0 (drop_att, common.cuh).  Read only by
  // the multi-head form, which takes the DROP instantiation iff drop_scale > 0.
  float drop_scale;
  SpmmEpilogue epi;   // the plain SpMM's store epilogue
};

enum { MODE_UNWEIGHTED = 0, MODE_WEIGHTED = 1, MODE_MULTIHEAD = 2, MODE_COMP_MULT = 3, MODE_COMP_SUB = 4 };
template <int MODE> constexpr bool is_comp_mode() { return MODE == MODE_COMP_MULT || MODE == MODE_COMP_SUB; }
// the shared-memory slab loop (stream_range_lean) serves the one-vector plain SpMM only
template <int MODE, int NV> constexpr bool is_lean() { return NV == 1 && (MODE == MODE_UNWEIGHTED || MODE == MODE_WEIGHTED); }
// Threads per block of every row-stream launch.  Measured on an H100 SXM (700 W), 128 vs 256, two alternating runs
// each: SpMM F=40 87 vs 90 us, arxiv / products F=128, mh-SpMM and the papers shard within 1 %; all outputs
// bit-identical.
constexpr int STREAM_BLOCK = 128;
enum { SRC_ONE = 0, SRC_TWO = 1, SRC_PEERS = 2 };
// What a launch_stream call runs: the plain SpMM (weighted iff p.val, any source form), its panel-major form, or
// the multi-head SpMM.
enum { FORM_PLAIN = 0, FORM_PANEL = 1, FORM_MULTIHEAD = 2 };
// What a store site of the plain SpMM writes: the sum (EPI_NONE), the residual epilogue of spmm_residual.cu
// (EPI_RESID), the label-propagation epilogue of label_prop.cu (EPI_LABELPROP), the residual epilogue with its b read
// on the device (gin.cu, EPI_RESID_DEV) or the accumulating epilogue of spmm_accum.cu (EPI_ACCUM, two stores per row).
enum { EPI_NONE = 0, EPI_RESID = 1, EPI_LABELPROP = 2, EPI_RESID_DEV = 3, EPI_ACCUM = 4 };
// EPI is the last template argument of the row kernel (spmm.cuh) and of stream_kernel.  cogdl_b200_last_kernel() names
// their instantiations spmm<tag>_kernel<...> and stream<tag>_kernel<...>, with the tag of their epilogue.
constexpr const char *EPI_TAG[] = {"", "_residual", "_labelprop", "_dcoef", "_accum"};

// The residual epilogue of one output element, rounded step by step as the unfused sequence
// `a * (r * spmm(x)) + b * z` rounds it (no contraction); r and z are used iff has_r / has_z.
__device__ __forceinline__ float residual_rn(float acc, float z, bool has_r, float r, bool has_z, float a, float b) {
  const float t = __fmul_rn(a, has_r ? __fmul_rn(r, acc) : acc);
  return has_z ? __fadd_rn(t, __fmul_rn(b, z)) : t;
}
__device__ __forceinline__ float2 residual_rn(float2 acc, float2 z, bool hr, float r, bool hz, float a, float b) {
  return make_float2(residual_rn(acc.x, z.x, hr, r, hz, a, b), residual_rn(acc.y, z.y, hr, r, hz, a, b));
}
__device__ __forceinline__ float4 residual_rn(float4 acc, float4 z, bool hr, float r, bool hz, float a, float b) {
  return make_float4(residual_rn(acc.x, z.x, hr, r, hz, a, b), residual_rn(acc.y, z.y, hr, r, hz, a, b),
                     residual_rn(acc.z, z.z, hr, r, hz, a, b), residual_rn(acc.w, z.w, hr, r, hz, a, b));
}

// acc of output row `row`, to be stored at yp (Z has Y's layout), with the residual epilogue of p (StreamParams or
// SpmmParams) applied.
template <typename VecT, typename P>
__device__ __forceinline__ VecT residual_out(const P &p, const VecT &acc, int64_t row, const VecT *yp) {
  const int64_t o = yp - reinterpret_cast<const VecT *>(p.Y);
  const bool hr = p.epi.row_scale != nullptr, hz = p.epi.Z != nullptr;
  const float r = hr ? __ldg(p.epi.row_scale + row) : 1.f;
  const VecT z = hz ? __ldg(reinterpret_cast<const VecT *>(p.epi.Z) + o) : vzero<VecT>();
  return residual_rn(acc, z, hr, r, hz, p.epi.res_a, p.epi.res_b);
}

// The residual epilogue with b = *res_b_dev, a coefficient that lives in device memory (GIN's 1 + eps, a trainable
// parameter), read by the kernel so the host never waits for it.  Only read when Z is given.
template <typename VecT, typename P>
__device__ __forceinline__ VecT residual_dev_out(const P &p, const VecT &acc, int64_t row, const VecT *yp) {
  const int64_t o = yp - reinterpret_cast<const VecT *>(p.Y);
  const bool hr = p.epi.row_scale != nullptr, hz = p.epi.Z != nullptr;
  const float r = hr ? __ldg(p.epi.row_scale + row) : 1.f;
  const VecT z = hz ? __ldg(reinterpret_cast<const VecT *>(p.epi.Z) + o) : vzero<VecT>();
  return residual_rn(acc, z, hr, r, hz, p.epi.res_a, hz ? __ldg(p.epi.res_b_dev) : 0.f);
}

// One element of the accumulating epilogue's running sum: fl(s + v), then times `scale` (fl) on the last hop -- what
// GRAND's `y.add_(x)` and the closing `y.div_(order + 1.0)` give on CUDA, where a division by a host scalar is a
// multiply by its fp32 reciprocal.
__device__ __forceinline__ float accum_rn(float s, float v, bool last, float scale) {
  const float t = __fadd_rn(s, v);
  return last ? __fmul_rn(t, scale) : t;
}
__device__ __forceinline__ float2 accum_rn(float2 s, float2 v, bool last, float scale) {
  return make_float2(accum_rn(s.x, v.x, last, scale), accum_rn(s.y, v.y, last, scale));
}
__device__ __forceinline__ float4 accum_rn(float4 s, float4 v, bool last, float scale) {
  return make_float4(accum_rn(s.x, v.x, last, scale), accum_rn(s.y, v.y, last, scale), accum_rn(s.z, v.z, last, scale),
                     accum_rn(s.w, v.w, last, scale));
}

// torch.clamp(v, lo, hi) as its CUDA kernel evaluates it: a NaN passes through, otherwise min(max(v, lo), hi) with the
// device fmaxf / fminf (so -0.0 against lo = 0 and lo > hi come out as torch gives them).
__device__ __forceinline__ float clamp_torch(float v, float lo, float hi) { return isnan(v) ? v : fminf(fmaxf(v, lo), hi); }
__device__ __forceinline__ float2 clamp_torch(float2 v, float lo, float hi) {
  return make_float2(clamp_torch(v.x, lo, hi), clamp_torch(v.y, lo, hi));
}
__device__ __forceinline__ float4 clamp_torch(float4 v, float lo, float hi) {
  return make_float4(clamp_torch(v.x, lo, hi), clamp_torch(v.y, lo, hi), clamp_torch(v.z, lo, hi), clamp_torch(v.w, lo, hi));
}

// The label-propagation epilogue of one output element: Z's element for a pinned row (the row reset of Correct &
// Smooth's fixed_post), else the residual epilogue, clamped when p.epi.has_clamp (autoscale_post).
template <typename VecT, typename P>
__device__ __forceinline__ VecT label_prop_out(const P &p, const VecT &acc, int64_t row, const VecT *yp) {
  if (p.epi.pin != nullptr && __ldg(p.epi.pin + row) != 0)
    return __ldg(reinterpret_cast<const VecT *>(p.epi.Z) + (yp - reinterpret_cast<const VecT *>(p.Y)));
  const VecT v = residual_out(p, acc, row, yp);
  return p.epi.has_clamp ? clamp_torch(v, p.epi.clamp_lo, p.epi.clamp_hi) : v;
}

// acc of output row `row`, to be stored at yp, with the epilogue EPI applied.
template <int EPI, typename VecT, typename P>
__device__ __forceinline__ VecT epilogue_out(const P &p, const VecT &acc, int64_t row, const VecT *yp) {
  if constexpr (EPI == EPI_RESID) return residual_out(p, acc, row, yp);
  else if constexpr (EPI == EPI_LABELPROP) return label_prop_out(p, acc, row, yp);
  else if constexpr (EPI == EPI_RESID_DEV) return residual_dev_out(p, acc, row, yp);
  else return acc;
}

// Pull one vector of ACC_in into the L1 ahead of its accumulating store (EPI_ACCUM).  Each element of ACC_in is read
// once per launch, by the thread that then writes ACC's element, so a line cached early holds current values for every
// element that will be read from it.  On a graph as small as Cora the SpMM runs a few dozen warps, each walking its
// rows one after the other, and the store's dependent load of ACC_in is the step's critical path; from the L1 it is
// short.
template <typename VecT>
__device__ __forceinline__ void prefetch_l1(const VecT *ptr) {
  asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr));
}

// Every store site of the plain SpMM: output row `row`'s finished acc, epilogue EPI applied, to yp.  The accumulating
// epilogue stores twice: the hop's row v = fl(r * acc) to yp (unless the last hop) and ACC's row fl(Z + v) in place.
// ACC's element is read and written by this thread only, and ACC is never gathered in the launch that writes it, so
// the plain load and the store cannot race.
template <int EPI, typename VecT, typename P>
__device__ __forceinline__ void epilogue_store(const P &p, const VecT &acc, int64_t row, VecT *yp) {
  if constexpr (EPI == EPI_ACCUM) {
    const int64_t o = yp - reinterpret_cast<const VecT *>(p.Y);
    const bool hr = p.epi.row_scale != nullptr;
    const VecT v = residual_rn(acc, vzero<VecT>(), hr, hr ? __ldg(p.epi.row_scale + row) : 1.f, false, 1.f, 0.f);
    if (!p.epi.acc_last) st_stream(yp, v);
    const VecT s = reinterpret_cast<const VecT *>(p.epi.Z)[o];
    st_stream(reinterpret_cast<VecT *>(p.epi.acc) + o, accum_rn(s, v, p.epi.acc_last != 0, p.epi.acc_scale));
  } else {
    st_stream(yp, epilogue_out<EPI>(p, acc, row, yp));
  }
}

// Stream the edge range [e, e_end).  ROWS: flush at row ends (segment); otherwise accumulate the
// whole range into acc (hub chunk).
template <typename VecT, int NV, int MODE, bool HAS_PERM, int SRC, int U, bool ROWS, bool PREFETCH, bool DROP = false,
          int EPI = EPI_NONE>
__device__ __forceinline__ void stream_range(const StreamParams &p, int e, const int e_end, const int cv,
                                             const bool (&colok)[NV], const int head, const int lane,
                                             VecT (&acc)[NV]) {
  const VecT *X0 = reinterpret_cast<const VecT *>(p.X0) + cv;
  const VecT *X1 = reinterpret_cast<const VecT *>(p.X1) + cv;
  VecT *Y = reinterpret_cast<VecT *>(p.Y) + cv;
  constexpr bool COMP = is_comp_mode<MODE>();
  const VecT *B = COMP ? reinterpret_cast<const VecT *>(p.B) + cv : nullptr;

  // slab registers: column, value / attention row / second index, owning row, owning row of the next edge
  int c = 0, rid = -1, rnx = -1, pe = 0;
  float v = 0.f;
  auto load_slab = [&](int base, int &c_, float &v_, int &pe_, int &rid_, int &rnx_) {
    const int q = base + lane;
    c_ = 0; v_ = 0.f; pe_ = 0; rid_ = -1; rnx_ = -1;
    if (q < e_end) {
      c_ = ld_stream(p.colind + q);
      if (MODE == MODE_WEIGHTED || COMP) v_ = ld_stream(p.val + q);
      if (MODE == MODE_MULTIHEAD) pe_ = HAS_PERM ? ld_stream(p.perm + q) : q;
      if (COMP) pe_ = ld_stream(p.idx2 + q);
      if (ROWS) {
        rid_ = ld_stream(p.hub.edge_row + q);
        if (q + 1 < e_end) rnx_ = __ldg(p.hub.edge_row + q + 1);
      }
    }
  };
  load_slab(e, c, v, pe, rid, rnx);

  for (; e < e_end; e += 32) {
    const int cnt = min(32, e_end - e);
    const unsigned endmask = ROWS ? __ballot_sync(FULL, lane < cnt && rid != rnx) : 0u;
    if constexpr (EPI == EPI_ACCUM && ROWS) {      // ACC_in of the rows that end in this slab, while its gathers run
      for (unsigned m = endmask; m != 0u; m &= m - 1u) {
        const int rj = __shfl_sync(FULL, rid, __ffs(m) - 1);
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (colok[k]) prefetch_l1(reinterpret_cast<const VecT *>(p.epi.Z) + cv + (int64_t)rj * p.ldv + k * 32);
      }
    }
    int cn, pn, ridn, rnxn;
    float vn;
    if (PREFETCH) load_slab(e + 32, cn, vn, pn, ridn, rnxn);  // next slab rides behind this slab's gathers

#pragma unroll 1
    for (int j = 0; j < cnt; j += U) {
      const bool full = (j + U <= cnt);
      const unsigned em = endmask >> j;
      VecT x[U][NV];
      VecT b[COMP ? U : 1][COMP ? NV : 1];
      float a[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int cj = __shfl_sync(FULL, c, j + u);
        const int pj = (MODE == MODE_MULTIHEAD || COMP) ? __shfl_sync(FULL, pe, j + u) : 0;
        if (full || j + u < cnt) {
          const VecT *xp;
          if (SRC == SRC_ONE || cj < p.n0) {
            xp = X0 + (int64_t)cj * p.ldv;
          } else if (SRC == SRC_TWO) {
            xp = X1 + ((int64_t)cj - p.n0) * p.ldv;
          } else {  // remote row: read it from the owner's HBM over NVLink
            const unsigned r = (unsigned)(cj - (int)p.n0);
            xp = reinterpret_cast<const VecT *>(p.peers[r >> p.peer_shift]) + cv +
                 (int64_t)(r & ((1u << p.peer_shift) - 1u)) * p.ldv;
          }
#pragma unroll
          for (int k = 0; k < NV; ++k)
            if (colok[k]) x[u][k] = ld_gather(xp + k * 32);
          if (MODE == MODE_MULTIHEAD && colok[0]) a[u] = __ldg(p.att + (int64_t)pj * p.H + head);
          if constexpr (COMP) {
            const VecT *bp = B + (int64_t)pj * p.ldv;
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) b[u][k] = ld_gather(bp + k * 32);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float vj = (MODE == MODE_WEIGHTED || COMP) ? __shfl_sync(FULL, v, j + u) : 0.f;
        const int rj = ROWS ? __shfl_sync(FULL, rid, j + u) : 0;
        if (full || j + u < cnt) {
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            if (colok[k]) {
              if (MODE == MODE_UNWEIGHTED) add_rn(acc[k], x[u][k]);          // 1.0f * x == x exactly
              else if (MODE == MODE_WEIGHTED) axpy_rn(acc[k], vj, x[u][k]);
              else if (MODE == MODE_COMP_MULT) axpy_rn(acc[k], vj, mul_rn(x[u][k], b[u][k]));
              else if (MODE == MODE_COMP_SUB) axpy_rn(acc[k], vj, sub_rn(x[u][k], b[u][k]));
              else axpy_rn(acc[k], DROP ? drop_att(a[u], p.drop_scale) : a[u], x[u][k]);
            }
          }
          if (ROWS && ((em >> u) & 1u)) {   // last edge of row rj: store and restart (warp-uniform)
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) {
                VecT *yp = Y + (int64_t)rj * p.ldv + k * 32;
                epilogue_store<EPI>(p, acc[k], rj, yp);
                acc[k] = vzero<VecT>();
              }
          }
        }
      }
    }
    if (PREFETCH) { c = cn; v = vn; pe = pn; rid = ridn; rnx = rnxn; }
    else load_slab(e + 32, c, v, pe, rid, rnx);
  }
}

// Lean form of stream_range for the plain SpMM (NV == 1, weighted / unweighted, any source form).  The
// general loop is issue-bound on the plain SpMM: three SHFL broadcasts per edge, each guarded by a BRA.DIV convergence check, and two
// predicate branches with BSSY/BSYNC pairs around every gather and every accumulate.  Here the slab
// (column, value, row) is parked in shared memory once (3 STS per 32 edges) and read back with broadcast LDS
// (no convergence requirement, column + value in ONE LDS.64), full batches run without per-edge predicates, and
// the row-end test is made once per batch on the ballot mask: ~15 instructions per edge.  Same accumulation
// order and rounding as stream_range (CSR order, separate fp32 multiply and add) => still bit-identical to
// the reference CPU loop on unsplit rows.  PF: the next slab's indices are loaded while this slab's gathers are
// in flight (3 more registers; the panel form's narrow gathers leave room for them).
//
// Row ends (ROWS).  The panel form (PF) finds them from rowptr: a row cursor r (the first row of the segment
// [r, r_end) whose end lies past the slab start) is kept in a register, lane k reads rowptr[r + k + 1], and every
// non-empty row whose end falls inside the slab sets its bit of the row-end mask.  That is one 128-byte line per slab,
// mostly re-read by the next slab, instead of edge_row's 4 bytes per edge (plus the neighbour's) in every pass.  The
// one-pass form keeps the edge_row test (`row != row of the next edge`, one ballot): there the cursor's longer
// dependent chain per slab costs more than the bytes it saves (SpMM F=40 +2 %, DESIGN 3.1).
template <typename VecT, int MODE, int SRC, int U, bool ROWS, bool PF = false, int EPI = EPI_NONE>
__device__ __forceinline__ void stream_range_lean(const StreamParams &p, int e, const int e_end, int r, const int r_end,
                                                  const int cv, const bool colok, const int lane, int2 *s_cv, int *s_r,
                                                  VecT &acc) {
  const VecT *X0 = reinterpret_cast<const VecT *>(p.X0) + cv;
  const VecT *X1 = reinterpret_cast<const VecT *>(p.X1) + cv;
  VecT *Y = reinterpret_cast<VecT *>(p.Y) + cv;
  auto src_ptr = [&](int cj) -> const VecT * {
    if (SRC == SRC_ONE || cj < p.n0) return X0 + (int64_t)cj * p.ldv;
    if (SRC == SRC_TWO) return X1 + ((int64_t)cj - p.n0) * p.ldv;
    const unsigned r = (unsigned)(cj - (int)p.n0);      // remote row: read it from the owner's HBM over NVLink
    return reinterpret_cast<const VecT *>(p.peers[r >> p.peer_shift]) + cv + (int64_t)(r & ((1u << p.peer_shift) - 1u)) * p.ldv;
  };
  auto accumulate = [&](float vj, const VecT &x) {
    if (MODE == MODE_UNWEIGHTED) add_rn(acc, x); else axpy_rn(acc, vj, x);
  };
  auto store_row = [&](int rj) {                    // row rj is complete: store it (epilogue applied) and restart
    VecT *yp = Y + (int64_t)rj * p.ldv;
    epilogue_store<EPI>(p, acc, rj, yp);
    acc = vzero<VecT>();
  };
  constexpr bool CURSOR = ROWS && PF;               // row ends from rowptr; otherwise (ROWS) from edge_row
  // column, value and (CURSOR) the end of row r + lane; INT_MAX past the segment's last row
  auto load_slab = [&](int base, int &c, float &v, int &end) {
    const int q = base + lane;
    c = 0; v = 0.f; end = INT_MAX;
    if (q < e_end) {
      c = ld_stream(p.colind + q);
      if (MODE == MODE_WEIGHTED) v = ld_stream(p.val + q);
    }
    if (CURSOR && base < e_end && r + lane < r_end) end = ld_stream(p.rowptr + r + lane + 1);
  };
  // Row-end mask of the slab [base, base + 32) from `end` (as load_slab left it), s_r[t] = the row whose last edge
  // is base + t, and r moved past every row that ends inside the slab.  A row is empty iff its end equals the end
  // of the row before; rows ending at or before base (empty rows at the segment's start) set no bit.  More than 32
  // rows can end inside one slab only through empty rows: then the next 32 are read.
  auto row_ends = [&](int base, int end) {
    unsigned mask = 0u;
    int end_before = base;
    for (;;) {
      int before = __shfl_up_sync(FULL, end, 1);
      if (lane == 0) before = end_before;
      const bool inside = end <= base + 32;
      const bool last_edge = inside && end > before;
      if (last_edge) s_r[end - 1 - base] = r + lane;
      mask |= __reduce_or_sync(FULL, last_edge ? 1u << (end - 1 - base) : 0u);
      const unsigned done = __ballot_sync(FULL, inside);   // a prefix of the lanes: ends do not decrease
      r += __popc(done);
      if (done != FULL) return mask;
      end_before = __shfl_sync(FULL, end, 31);
      end = r + lane < r_end ? ld_stream(p.rowptr + r + lane + 1) : INT_MAX;
    }
  };
  int pc = 0, pend = INT_MAX;                       // PF: the slab loaded one iteration ahead
  float pv = 0.f;
  if (PF) load_slab(e, pc, pv, pend);
  for (; e < e_end; e += 32) {
    const int cnt = min(32, e_end - e);
    const int q = e + lane;
    int c, end, rid = -1, rnx = -1;
    float v;
    if (PF) { c = pc; v = pv; end = pend; }
    else load_slab(e, c, v, end);
    if (ROWS && !CURSOR && q < e_end) {
      rid = ld_stream(p.hub.edge_row + q);
      if (q + 1 < e_end) rnx = __ldg(p.hub.edge_row + q + 1);
    }
    unsigned endmask = ROWS && !CURSOR ? __ballot_sync(FULL, lane < cnt && rid != rnx) : 0u;
    __syncwarp();                                   // everybody is done reading the previous slab
    s_cv[lane] = make_int2(c, __float_as_int(v));
    if (CURSOR) endmask = row_ends(e, end);
    else if (ROWS) s_r[lane] = rid;
    __syncwarp();
    if constexpr (EPI == EPI_ACCUM && ROWS) {      // ACC_in of the rows that end in this slab, while its gathers run
      for (unsigned m = endmask; m != 0u; m &= m - 1u)
        if (colok) prefetch_l1(reinterpret_cast<const VecT *>(p.epi.Z) + cv + (int64_t)s_r[__ffs(m) - 1] * p.ldv);
    }
    if (PF) load_slab(e + 32, pc, pv, pend);        // consumed by the next iteration only (r is already past this slab)
    int j = 0;
#pragma unroll 1
    for (; j + U <= cnt; j += U) {                  // full batches: no per-edge predicates
      int2 cw[U];
      VecT x[U];
      // PF: the values are read back when consumed, not with the columns, so a deep batch does not hold U of
      // them across the gathers (at U = 8 that is the difference between spilling and not)
      auto val_of = [&](int u) {
        return __int_as_float(PF ? reinterpret_cast<const volatile int *>(s_cv + j + u)[1] : cw[u].y);
      };
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (PF) cw[u].x = s_cv[j + u].x;                          // broadcast LDS
        else cw[u] = s_cv[j + u];                                 // broadcast LDS.64
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (colok) x[u] = ld_gather(src_ptr(cw[u].x));
      const unsigned em = ROWS ? ((endmask >> j) & ((1u << U) - 1u)) : 0u;
      if (em == 0u) {                               // no row ends inside this batch
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (colok) accumulate(val_of(u), x[u]);
      } else {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (colok) accumulate(val_of(u), x[u]);
          if ((em >> u) & 1u) {                     // last edge of its row: store and restart (warp-uniform)
            const int rj = s_r[j + u];
            if (colok) store_row(rj);
          }
        }
      }
    }
#pragma unroll 1
    for (; j < cnt; ++j) {                          // tail of the last slab: one edge at a time
      const int2 cw = s_cv[j];
      if (colok) accumulate(__int_as_float(cw.y), ld_gather(src_ptr(cw.x)));
      if (ROWS && ((endmask >> j) & 1u)) {
        const int rj = s_r[j];
        if (colok) store_row(rj);
      }
    }
  }
}

// One work item processed by one warp: wid = item * S + slice (multi-head), slice = blockIdx.y (PANEL).
template <typename VecT, int NV, int MODE, bool HAS_PERM, int SRC, int U, bool PREFETCH, bool PANEL, bool DROP = false,
          int EPI = EPI_NONE>
__device__ __forceinline__ void stream_item(const StreamParams &p, const int64_t wid, const int lane, int2 *s_cv, int *s_r) {
  constexpr int TILE = 32 * NV;
  constexpr bool SLICED = (MODE == MODE_MULTIHEAD || PANEL);
  int64_t item = wid;
  int slice = PANEL ? (int)blockIdx.y : 0;
  if (MODE == MODE_MULTIHEAD) { item = wid / p.S; slice = (int)(wid - item * p.S); }
  VecT *Y = reinterpret_cast<VecT *>(p.Y);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);
  constexpr bool LEAN = is_lean<MODE, NV>();

  // column tiles: the multi-head and panel forms own exactly one 32-vector slice; the plain form loops over
  // the row in TILE-vector passes (one pass for F <= 128 * NV)
  const int t_begin = SLICED ? slice * 32 : 0;
  const int t_end = SLICED ? t_begin + 1 : p.ldv;

  if (item < p.hub.n_chunks) {
    const WorkItem w = decode_item(item, 0, p.rowptr, p.hub);
    for (int tile0 = t_begin; tile0 < t_end; tile0 += TILE) {
      const int cv = tile0 + lane;
      bool colok[NV];
      VecT acc[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) { colok[k] = (cv + k * 32) < p.ldv; acc[k] = vzero<VecT>(); }
      const int head = (MODE == MODE_MULTIHEAD && colok[0]) ? cv / p.FVL : 0;
      if constexpr (LEAN) stream_range_lean<VecT, MODE, SRC, U, false, PANEL && PREFETCH>(p, w.lb, w.hb, 0, 0, cv, colok[0], lane, s_cv, s_r, acc[0]);
      else stream_range<VecT, NV, MODE, HAS_PERM, SRC, U, false, PREFETCH, DROP>(p, w.lb, w.hb, cv, colok, head, lane, acc);
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (colok[k]) st_cg(P + (int64_t)w.slot * p.ldv + cv + k * 32, acc[k]);
    }
    // multi-head: every slice of every chunk arrives at the row's counter and the last one combines the whole
    // row.  Panel mode: one counter per (row, panel) at counters[panel * n_chunks + first], and the last chunk of
    // the panel combines just its 32 vectors -- the row's last arrival overall would come in the last panel,
    // which would turn a long hub's merge into an end-of-kernel tail.
    WorkItem wa = w;
    if (MODE == MODE_MULTIHEAD) wa.n_row_chunks = w.n_row_chunks * p.S;
    bool last;
    if constexpr (PANEL) {
      HubView hv = p.hub;
      hv.counters += (int64_t)slice * p.hub.n_chunks;
      last = hub_arrive_last<32>(wa, hv, lane);
    } else {
      last = hub_arrive_last<32>(wa, p.hub, lane);
    }
    if (last) {
      const int c_begin = PANEL ? t_begin : 0, c_end = PANEL ? min(t_begin + 32, p.ldv) : p.ldv;
      for (int cv = c_begin + lane; cv < c_end; cv += 32) {
        const VecT *pp = P + (int64_t)w.first * p.ldv + cv;
        const VecT s = merge_chunks<8>(w.n_row_chunks, [&](int q) { return ld_cg(pp + (int64_t)q * p.ldv); },
                                       [](VecT &a, const VecT &t) { add_rn(a, t); });
        VecT *yp = Y + (int64_t)w.row * p.ldv + cv;
        epilogue_store<EPI>(p, s, w.row, yp);
      }
    }
    return;
  }

  const int64_t seg = item - p.hub.n_chunks;
  if (seg >= p.hub.n_segs) return;
  const int2 rr = __ldg(p.hub.segs + seg);
  const int e_begin = __ldg(p.rowptr + rr.x), e_end = __ldg(p.rowptr + rr.y);

  for (int tile0 = t_begin; tile0 < t_end; tile0 += TILE) {
    const int cv = tile0 + lane;
    bool colok[NV];
    VecT acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) { colok[k] = (cv + k * 32) < p.ldv; acc[k] = vzero<VecT>(); }
    const int head = (MODE == MODE_MULTIHEAD && colok[0]) ? cv / p.FVL : 0;
    if (p.hub.n_empty_rows > 0) {
      // rows without edges never show up in the edge stream: zero-fill them here
      for (int rb = rr.x; rb < rr.y; rb += 32) {
        const int row = rb + lane;
        unsigned m = __ballot_sync(FULL, row < rr.y && __ldg(p.rowptr + row + 1) == __ldg(p.rowptr + row));
        while (m) {
          const int k0 = __ffs(m) - 1;
          m &= m - 1;
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            if (colok[k]) {
              VecT *yp = Y + (int64_t)(rb + k0) * p.ldv + cv + k * 32;
              epilogue_store<EPI>(p, vzero<VecT>(), rb + k0, yp);
            }
          }
        }
      }
    }
    if constexpr (LEAN) stream_range_lean<VecT, MODE, SRC, U, true, PANEL && PREFETCH, EPI>(p, e_begin, e_end, rr.x, rr.y, cv, colok[0], lane, s_cv, s_r, acc[0]);
    else stream_range<VecT, NV, MODE, HAS_PERM, SRC, U, true, PREFETCH, DROP, EPI>(p, e_begin, e_end, cv, colok, head, lane, acc);
  }
}

template <typename VecT, int NV, int MODE, bool HAS_PERM, int SRC, int U, int MINB, bool PREFETCH, bool PANEL = false,
          bool DROP = false, int EPI = EPI_NONE>
__global__ void __launch_bounds__(256, MINB) stream_kernel(const StreamParams p) {
  const int lane = threadIdx.x & 31;
  constexpr bool LEAN = is_lean<MODE, NV>();
  __shared__ int2 s_cv_all[LEAN ? 8 : 1][32];
  __shared__ int s_r_all[LEAN ? 8 : 1][32];
  int2 *s_cv = s_cv_all[LEAN ? (threadIdx.x >> 5) : 0];
  int *s_r = s_r_all[LEAN ? (threadIdx.x >> 5) : 0];
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  stream_item<VecT, NV, MODE, HAS_PERM, SRC, U, PREFETCH, PANEL, DROP, EPI>(p, wid, lane, s_cv, s_r);
}

// Launch helper: picks the instantiation of FORM for (weighted, perm, source form); U / MINB fixed by the caller.
// The panel form has p.S panels of 32 VecT each (grid.y); the multi-head form p.S slices per item.  EPI: the store
// epilogue of the plain or panel form, which then reads one source.
template <typename VecT, int NV, int U, int MINB, bool PREFETCH = true, int FORM = FORM_PLAIN, int EPI = EPI_NONE>
static int launch_stream(const StreamParams &p, cudaStream_t stream) {
  static_assert(FORM == FORM_PLAIN || NV == 1, "the panel and multi-head forms have one VecT per lane");
  static_assert(EPI == EPI_NONE || FORM != FORM_MULTIHEAD, "the store epilogues are forms of the plain SpMM");
  const int64_t warps = ((int64_t)p.hub.n_chunks + p.hub.n_segs) * (FORM == FORM_MULTIHEAD ? p.S : 1);
  // Threads per block: a launch parameter only -- the kernel indexes its per-warp slabs by warp-in-block and takes its
  // item from the global warp index, so every block size runs the same SASS and gives the same bits.  A block's warp
  // slots go to the next block only when its SLOWEST warp has retired; item durations spread (gathers that miss L2,
  // hub merges), so smaller blocks keep more warp slots busy -- most visibly for the two-vectors-per-lane
  // instantiation (F = 256).  A persistent form (grid = resident warp slots, items drawn from a ticket counter in the
  // plan) was also built and measured slower (the ticket loop needs 64 registers = 32 warps/SM) -- removed.
  const int64_t blocks = ceil_div(warps * 32, STREAM_BLOCK);
  if (blocks == 0) return COGDL_B200_OK;
  if (blocks > 0x7fffffffLL) return set_error(COGDL_B200_EINVAL, "stream kernel: problem too large for one launch");
  const dim3 grid((unsigned)blocks, FORM == FORM_PANEL ? (unsigned)p.S : 1u);
  const int src = p.n_peers > 0 ? SRC_PEERS : (p.n0 != INT64_MAX ? SRC_TWO : SRC_ONE);
  if ((FORM != FORM_PLAIN || EPI != EPI_NONE) && src != SRC_ONE)
    return set_error(COGDL_B200_EINVAL, "stream kernel: the panel, multi-head and epilogue forms read one source");
  const bool drop = FORM == FORM_MULTIHEAD && p.drop_scale > 0.f;
  note_kernel("cogdl_b200::stream%s_kernel<%s,NV=%d,%s%s%s,%s,U=%d,MINB=%d%s>", EPI_TAG[EPI],
              sizeof(VecT) == 16 ? "float4" : (sizeof(VecT) == 8 ? "float2" : "float"), NV,
              FORM == FORM_MULTIHEAD ? "multihead" : (p.val ? "weighted" : "unweighted"),
              (FORM == FORM_MULTIHEAD && p.perm) ? "+perm" : "", drop ? "+drop" : "",
              src == SRC_PEERS ? "SRC_PEERS" : (src == SRC_TWO ? "SRC_TWO" : "SRC_ONE"), U, MINB,
              PREFETCH ? ",prefetch" : "");
  if (FORM == FORM_PANEL && p.S > 1) append_kernel_note(",panels=%d", p.S);
  append_kernel_note(" block=%d", STREAM_BLOCK);
  if constexpr (FORM == FORM_MULTIHEAD) {
    if (drop) {
      if (p.perm) stream_kernel<VecT, 1, MODE_MULTIHEAD, true, SRC_ONE, U, MINB, PREFETCH, false, true><<<grid, STREAM_BLOCK, 0, stream>>>(p);
      else stream_kernel<VecT, 1, MODE_MULTIHEAD, false, SRC_ONE, U, MINB, PREFETCH, false, true><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    } else if (p.perm) {
      stream_kernel<VecT, 1, MODE_MULTIHEAD, true, SRC_ONE, U, MINB, PREFETCH><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    } else {
      stream_kernel<VecT, 1, MODE_MULTIHEAD, false, SRC_ONE, U, MINB, PREFETCH><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    }
  } else if constexpr (FORM == FORM_PANEL) {
    if (p.val) stream_kernel<VecT, 1, MODE_WEIGHTED, false, SRC_ONE, U, MINB, PREFETCH, true, false, EPI><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    else stream_kernel<VecT, 1, MODE_UNWEIGHTED, false, SRC_ONE, U, MINB, PREFETCH, true, false, EPI><<<grid, STREAM_BLOCK, 0, stream>>>(p);
  } else if (src == SRC_ONE) {
    if (p.val) stream_kernel<VecT, NV, MODE_WEIGHTED, false, SRC_ONE, U, MINB, PREFETCH, false, false, EPI><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    else stream_kernel<VecT, NV, MODE_UNWEIGHTED, false, SRC_ONE, U, MINB, PREFETCH, false, false, EPI><<<grid, STREAM_BLOCK, 0, stream>>>(p);
  } else if constexpr (EPI == EPI_NONE) {       // the two-source and peer forms have no epilogue (turned away above)
    if (p.val) {
      if (src == SRC_PEERS) stream_kernel<VecT, NV, MODE_WEIGHTED, false, SRC_PEERS, U, MINB, PREFETCH><<<grid, STREAM_BLOCK, 0, stream>>>(p);
      else stream_kernel<VecT, NV, MODE_WEIGHTED, false, SRC_TWO, U, MINB, PREFETCH><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    } else {
      if (src == SRC_PEERS) stream_kernel<VecT, NV, MODE_UNWEIGHTED, false, SRC_PEERS, U, MINB, PREFETCH><<<grid, STREAM_BLOCK, 0, stream>>>(p);
      else stream_kernel<VecT, NV, MODE_UNWEIGHTED, false, SRC_TWO, U, MINB, PREFETCH><<<grid, STREAM_BLOCK, 0, stream>>>(p);
    }
  }
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

}  // namespace cogdl_b200

// spmm.cuh -- the fp32 SpMM's sub-warp row kernel, its dispatch by width, alignment, plan form and panel count, and
// the host entry in front of it, shared by the plain SpMM (spmm.cu), the SpMM with a residual epilogue
// (spmm_residual.cu), the label-propagation step (label_prop.cu), the GIN aggregation (gin.cu) and GRAND's propagation
// hop (spmm_accum.cu).  EPI, the last template argument of the row kernel and of stream_kernel, selects the epilogue:
// every finished row is written by epilogue_store<EPI> (stream.cuh) -- acc itself for EPI_NONE -- with the operands in
// SpmmEpilogue.  Design notes: spmm.cu.
#pragma once
#include "common.cuh"
#include "stream.cuh"

namespace cogdl_b200 {

struct SpmmParams {
  const float *peers[8] = {};
  int n_peers = 0;
  int peer_shift = 0;
  const int *rowptr;
  const int *colind;
  const float *val;
  const float *X0;
  const float *X1;
  int64_t n0 = INT64_MAX;  // columns < n0 read X0, others X1[c - n0]
  float *Y;
  int64_t n_rows;
  int FV;      // feature row length in VecT units
  HubView hub;
  SpmmEpilogue epi;   // the store epilogue (stream.cuh)
};

template <typename VecT, int GROUP, int NV, bool HAS_VAL, int EPI>
__device__ __forceinline__ void spmm_rows(const SpmmParams &p) {
  constexpr int U0 = (NV == 1) ? 8 : (NV == 2 ? 4 : 2);
  constexpr int U = U0 < GROUP ? U0 : GROUP;
  constexpr int TILE = GROUP * NV;  // vector columns covered per pass
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t item = tid / GROUP;
  const WorkItem w = decode_item(item, p.n_rows, p.rowptr, p.hub);
  const bool warp_has_chunk = (tid - lane) / GROUP < p.hub.n_chunks;  // warp-uniform

  const VecT *X0 = reinterpret_cast<const VecT *>(p.X0);
  const VecT *X1 = reinterpret_cast<const VecT *>(p.X1);
  VecT *Y = reinterpret_cast<VecT *>(p.Y);
  VecT *P = reinterpret_cast<VecT *>(p.hub.partials);

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);  // keep loop trip counts warp-uniform for the shuffles

  // Feature rows wider than one pass (F > 256 on the vector path) are covered by looping over
  // column tiles inside the warp (indices are re-read per tile, as the reference's grid.y tiles do).
  for (int tile0 = 0; tile0 < p.FV; tile0 += TILE) {
    const int cv = tile0 + gl;  // this lane's first vector column in this tile
    bool colok[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) colok[k] = (cv + k * GROUP) < p.FV;
    VecT acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = vzero<VecT>();
    if constexpr (EPI == EPI_ACCUM) {              // ACC_in of this row, ahead of its store (prefetch_l1, stream.cuh)
      if (!w.is_chunk && w.active) {
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (colok[k]) prefetch_l1(reinterpret_cast<const VecT *>(p.epi.Z) + (int64_t)w.row * p.FV + cv + k * GROUP);
      }
    }

    int c = 0;
    float v = 0.f;
    {
      const int e = w.lb + gl;
      if (e < w.hb) {
        c = ld_stream(p.colind + e);
        v = HAS_VAL ? ld_stream(p.val + e) : 1.f;
      }
    }
    for (int off = 0; off < maxdeg; off += GROUP) {
      const int cnt = min(GROUP, w.hb - w.lb - off);  // <= 0 for groups whose row is already done
      int cn = 0;
      float vn = 0.f;
      {
        const int e = w.lb + off + GROUP + gl;  // prefetch the next index/value slab
        if (e < w.hb) {
          cn = ld_stream(p.colind + e);
          vn = HAS_VAL ? ld_stream(p.val + e) : 1.f;
        }
      }
#pragma unroll 1
      for (int j = 0; j < GROUP; j += U) {
        if (GROUP == 32) {
          if (j >= cnt) break;
        } else {
          if (!__any_sync(FULL, j < cnt)) break;
        }
        VecT x[U][NV];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, c, j + u, GROUP);
          if (j + u < cnt) {
            const VecT *xp = (cj < p.n0) ? X0 + (int64_t)cj * p.FV : X1 + ((int64_t)cj - p.n0) * p.FV;
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) x[u][k] = ld_gather(xp + cv + k * GROUP);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float vj = __shfl_sync(FULL, v, j + u, GROUP);
          if (j + u < cnt) {
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (colok[k]) axpy_rn(acc[k], vj, x[u][k]);
          }
        }
      }
      c = cn;
      v = vn;
    }

    if (!w.is_chunk) {
      if (w.active) {
        VecT *yp = Y + (int64_t)w.row * p.FV + cv;
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (colok[k]) epilogue_store<EPI>(p, acc[k], w.row, yp + k * GROUP);
      }
    } else {
      VecT *pp = P + (int64_t)w.slot * p.FV + cv;
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (colok[k]) st_cg(pp + k * GROUP, acc[k]);
    }
  }

  if (warp_has_chunk) {
    if (hub_arrive_last<GROUP>(w, p.hub, gl)) {
      // combine this row's partial sums in chunk order (deterministic, independent of arrival)
      for (int cv = gl; cv < p.FV; cv += GROUP) {
        const VecT *pp = P + (int64_t)w.first * p.FV + cv;
        const VecT s = merge_chunks<1>(w.n_row_chunks, [&](int q) { return ld_cg(pp + (int64_t)q * p.FV); },
                                       [](VecT &a, const VecT &t) { add_rn(a, t); });
        VecT *yp = Y + (int64_t)w.row * p.FV + cv;
        epilogue_store<EPI>(p, s, w.row, yp);
      }
    }
  }
}

// EPI_NONE leaves the register budget to ptxas.  The epilogues ask for at least 3 blocks per SM: left to itself ptxas
// fits the GROUP=4 float4 weighted residual instantiation in 64 registers and spills; 80 registers hold every
// instantiation without spilling.
template <typename VecT, int GROUP, int NV, bool HAS_VAL, int EPI>
__global__ void __launch_bounds__(256, EPI == EPI_NONE ? 0 : 3) spmm_kernel(const SpmmParams p) {
  spmm_rows<VecT, GROUP, NV, HAS_VAL, EPI>(p);
}

// ------------------------------------------------------------------------------------------
// Row-stream form (stream.cuh), used whenever the plan carries segments and a full warp owns the
// row (F >= 68, or >= 17 on the scalar path).
// ------------------------------------------------------------------------------------------
static StreamParams to_stream(const SpmmParams &p) {
  StreamParams q;
  q.rowptr = p.rowptr; q.colind = p.colind; q.val = p.val; q.att = nullptr; q.perm = nullptr;
  q.X0 = p.X0; q.X1 = p.X1; q.n0 = p.n0; q.Y = p.Y; q.ldv = p.FV; q.H = 1; q.FVL = p.FV; q.S = 1;
  q.hub = p.hub;
  q.n_peers = p.n_peers; q.peer_shift = p.peer_shift;
  for (int i = 0; i < 8; ++i) q.peers[i] = p.peers[i];
  q.epi = p.epi;
  return q;
}

template <typename VecT, int NV, int EPI>
static int launch_spmm_stream(const SpmmParams &p, cudaStream_t stream) {
  const StreamParams q = to_stream(p);
  if constexpr (NV == 1 && sizeof(VecT) == 16) {
    // lean loop (stream_range_lean), U=4, 48 registers (40 warps/SM); the epilogue's Z row needs 4 more registers
    // than that budget holds, so the epilogue forms run at 32 warps/SM rather than spill
    return launch_stream<VecT, 1, 4, EPI != EPI_NONE ? 4 : 5, false, FORM_PLAIN, EPI>(q, stream);
  } else {
    constexpr int U = (NV == 1) ? 8 : (NV == 2 ? 4 : 2);
    return launch_stream<VecT, NV, U, 1, true, FORM_PLAIN, EPI>(q, stream);
  }
}

// ------------------------------------------------------------------------------------------
// Panel mode.  With uniformly random columns a gathered X row survives in the L2 only if it is reused before
// ~L2-size of other traffic evicts it; once X outgrows the L2 most gathers go to DRAM.  P passes over the graph,
// pass p gathering only columns [p*F/P, (p+1)*F/P) (panel-major grid, stream.cuh), keep the live panel
// L2-resident so X comes from DRAM about once.  Every lane owns one VecT of the panel (F/P = 32, 64 or 128
// floats => float, float2, float4); accumulation order per element is unchanged, so the output is
// bit-identical to P = 1.
// ------------------------------------------------------------------------------------------
static int64_t device_l2_bytes() {
  static int cache[64] = {0};   // per device; racing first calls store the same value
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  if (cache[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev) != cudaSuccess || v <= 0) return 0;
    cache[dev] = v;
  }
  return cache[dev];
}

// Largest share of the L2 one panel of X may take.  7/8 picks 64-float panels on the arxiv shape (F = 128 -> P = 2,
// F = 256 -> P = 4; 43 MB panels in the 50 MB L2), the fastest measured (DESIGN 3.1): 32-float panels (P = 4 at
// F = 128) keep X in the L2 better still, but their one-float lanes cost more issue slots than the misses they save.
constexpr int64_t PANEL_THETA_NUM = 7, PANEL_THETA_DEN = 8;

// A panel is exactly 32 lanes x one VecT: F / P must be 32, 64 or 128 floats (a 96-float panel would leave a
// partial VecT tile that the launch below does not have).
static bool panel_width_ok(int64_t F, int P) {
  if (P < 1 || P > COGDL_B200_MAX_PANELS || F % P != 0) return false;
  const int64_t w = F / P;
  return w == 32 || w == 64 || w == 128;
}

// Smallest power of two P whose panel fits the budget; 1 when X already fits or even the narrowest panels
// do not (then the extra index passes cost more than the misses they save).
static int auto_panels(int64_t x_rows, int64_t F) {
  const int64_t x_bytes = x_rows * F * (int64_t)sizeof(float);
  const int64_t budget = device_l2_bytes() * PANEL_THETA_NUM / PANEL_THETA_DEN;
  if (budget <= 0 || x_bytes <= budget) return 1;
  for (int P = 2; P <= COGDL_B200_MAX_PANELS && 32 * (int64_t)P <= F; P *= 2)
    if (panel_width_ok(F, P) && x_bytes / P <= budget) return P;
  return 1;
}

template <int EPI>
static int launch_spmm_panels(const SpmmParams &p, int64_t F, int P, cudaStream_t stream) {
  StreamParams q = to_stream(p);
  q.S = P;
  switch (F / P) {
    case 32:
      q.ldv = q.FVL = (int)F;
      return launch_stream<float, 1, 8, 6, true, FORM_PANEL, EPI>(q, stream);
    case 64:
      // the device coefficient's load costs the weighted 64-float panel loop one register more than 5 blocks per SM
      // leave it (48), so that epilogue runs at 4 rather than spill
      q.ldv = q.FVL = (int)(F / 2);
      return launch_stream<float2, 1, 8, EPI == EPI_RESID_DEV ? 4 : 5, true, FORM_PANEL, EPI>(q, stream);
    default:
      q.ldv = q.FVL = (int)(F / 4);
      return launch_stream<float4, 1, 4, EPI != EPI_NONE ? 4 : 5, true, FORM_PANEL, EPI>(q, stream);
  }
}

// the row kernel's name in its launch errors, per epilogue
constexpr const char *EPI_WHO[] = {"spmm", "spmm_residual", "label_prop", "spmm_dcoef", "spmm_accum"};

template <typename VecT, int GROUP, int NV, int EPI>
static int launch_spmm(const SpmmParams &p, cudaStream_t stream) {
  return launch_items(p.val ? spmm_kernel<VecT, GROUP, NV, true, EPI> : spmm_kernel<VecT, GROUP, NV, false, EPI>, p,
                      (int64_t)p.hub.n_chunks + p.n_rows, GROUP, stream, EPI_WHO[EPI],
                      "cogdl_b200::spmm%s_kernel<%s,GROUP=%d,NV=%d,%s>", EPI_TAG[EPI],
                      sizeof(VecT) == 16 ? "float4" : "float", GROUP, NV, p.val ? "weighted" : "unweighted");
}

// narrow rows (F = 40 -> 10 float4): the lean row-stream form with the idle lanes masked beats the sub-warp
// row kernel once a row needs at least this many vectors
constexpr int SPMM_STREAM_MIN_FV = 9;

template <typename VecT, int EPI>
static int dispatch_spmm(const SpmmParams &p, cudaStream_t s) {
  const int fv = p.FV;
  // peer form: only the row-stream kernel decodes (owner << shift | row) columns (SRC_PEERS); the
  // sub-warp row kernel below would read them as X1[c - n0].  NV = 1 masks lanes >= fv.
  if (p.n_peers > 0 && fv <= 32) return launch_spmm_stream<VecT, 1, EPI>(p, s);
  const bool stream = p.hub.n_segs > 0;
  if (stream && fv >= SPMM_STREAM_MIN_FV && fv <= 16) return launch_spmm_stream<VecT, 1, EPI>(p, s);
  if (fv <= 1) return launch_spmm<VecT, 1, 1, EPI>(p, s);
  if (fv <= 2) return launch_spmm<VecT, 2, 1, EPI>(p, s);
  if (fv <= 4) return launch_spmm<VecT, 4, 1, EPI>(p, s);
  if (fv <= 8) return launch_spmm<VecT, 8, 1, EPI>(p, s);
  if (fv <= 16) return launch_spmm<VecT, 16, 1, EPI>(p, s);
  if (fv <= 32) return stream ? launch_spmm_stream<VecT, 1, EPI>(p, s) : launch_spmm<VecT, 32, 1, EPI>(p, s);
  if constexpr (sizeof(VecT) == 4) {
    if (fv > 64) return stream ? launch_spmm_stream<VecT, 4, EPI>(p, s) : launch_spmm<VecT, 32, 4, EPI>(p, s);
  }
  return stream ? launch_spmm_stream<VecT, 2, EPI>(p, s) : launch_spmm<VecT, 32, 2, EPI>(p, s);
}

// [p, p + n) and [q, q + m) share a byte
static inline bool overlaps(const float *p, int64_t n, const float *q, int64_t m) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
  return a < b + (uintptr_t)m * sizeof(float) && b < a + (uintptr_t)n * sizeof(float);
}

// The output checks of the epilogue entries, for a non-empty output `out` ([n_rows, F], `name` in the messages): the
// kernels read X, Z and row_scale (read-only cache path) while other warps write finished rows of out, so out may
// overlap none of them.  X holds x_rows rows (colind < x_rows), so an empty X can only coincide with out.  Z and
// row_scale are optional.
static int check_output_apart(const char *who, const char *name, const float *out, int64_t n_rows, int64_t F,
                              const float *X, int64_t x_rows, const float *Z, const float *row_scale) {
  const int64_t nf = n_rows * F;
  CB_REQUIRE(out != X && !overlaps(out, nf, X, x_rows * F), "%s: %s overlaps X", who, name);
  CB_REQUIRE(!Z || !overlaps(out, nf, Z, nf), "%s: %s overlaps Z", who, name);
  CB_REQUIRE(!row_scale || !overlaps(out, nf, row_scale, n_rows), "%s: %s overlaps row_scale", who, name);
  return COGDL_B200_OK;
}

// The host side of every fp32 SpMM entry point: argument checks, the parameters, the panel count and the dispatch.
// X1 (nullptr = X0) serves the columns >= n0 (two-source form); peers are the peer form's shards; epi holds the
// operands of the epilogue EPI (stream.cuh).  x_rows, X0's row count, sizes the automatic panel count (panels = 0).
// Static, so each object instantiates only the form it calls.
template <int EPI>
static int spmm_entry(const int32_t *rowptr, const int32_t *colind, const float *val, const float *X0, int64_t n0,
                      const float *X1, float *Y, int64_t n_rows, int64_t F, const cogdl_b200_hub_plan_t *plan,
                      cogdl_b200_stream_t stream, const char *who, const float *const *peers = nullptr,
                      int n_peers = 0, int peer_shift = 0, int64_t x_rows = 0, int panels = 1,
                      const SpmmEpilogue &epi = {}) {
  CB_REQUIRE(n_rows >= 0 && F >= 0, "%s: negative size (n_rows=%lld, F=%lld)", who, (long long)n_rows, (long long)F);
  CB_REQUIRE(x_rows >= 0 && panels >= 0, "%s: negative x_rows / panels", who);
  if (n_rows == 0 || F == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && X0 && Y, "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && F < 0x7fffffffLL, "%s: n_rows / F must fit int32", who);
  int rc = check_plan(plan, cogdl_b200_spmm_scratch_bytes(plan ? plan->n_chunks : 0, F));
  if (rc) return rc;
  SpmmParams p;
  p.rowptr = rowptr; p.colind = colind; p.val = val; p.X0 = X0; p.X1 = X1 ? X1 : X0; p.n0 = n0;
  p.Y = Y; p.n_rows = n_rows; p.hub = hub_view(plan);
  p.n_peers = n_peers; p.peer_shift = peer_shift;
  p.epi = epi;
  bool peers_aligned = true;
  for (int i = 0; i < n_peers; ++i) {
    p.peers[i] = peers[i];
    peers_aligned = peers_aligned && aligned16(peers[i]);
  }
  if (n_peers > 0)
    CB_REQUIRE(p.hub.n_segs > 0 && F % 4 == 0 && F <= 512 && peers_aligned && aligned16(X0) && aligned16(Y),
               "%s: the peer form needs a plan with segments, F %% 4 == 0, F <= 512 and 16-byte aligned buffers", who);
  const bool vec = (F % 4 == 0) && aligned16(X0) && aligned16(p.X1) && aligned16(Y) && aligned16(epi.Z) &&
                   aligned16(epi.acc) && (p.hub.n_chunks == 0 || aligned16(p.hub.partials));
  if (vec) p.FV = (int)(F / 4);
  const bool panel_form = vec && n_peers == 0 && n0 == INT64_MAX && p.hub.n_segs > 0 && F % 32 == 0;
  if (panels > 1)
    CB_REQUIRE(panel_form && panel_width_ok(F, panels),
               "%s: %d panels need a plan with segments, one source, 16-byte aligned buffers and F / panels in "
               "{32, 64, 128} (F=%lld, at most %d panels)", who, panels, (long long)F, COGDL_B200_MAX_PANELS);
  const int P = panels == 0 ? (panel_form ? auto_panels(x_rows, F) : 1) : panels;
  if (P > 1) return launch_spmm_panels<EPI>(p, F, P, (cudaStream_t)stream);
  if (vec) return dispatch_spmm<float4, EPI>(p, (cudaStream_t)stream);
  p.FV = (int)F;
  return dispatch_spmm<float, EPI>(p, (cudaStream_t)stream);
}

}  // namespace cogdl_b200

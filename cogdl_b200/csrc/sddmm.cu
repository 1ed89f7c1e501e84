// sddmm.cu -- CSR SDDMM and multi-head SDDMM for sm_90a.
//
//   sddmm   : out[p]   = < D1[row(p), :],    D2[colind[p], :]    >           (NSEG = 1)
//   mhsddmm : out[p,h] = < grad[row(p),h,:], feat[colind[p],h,:] >           (NSEG = H)
//
// Replaces sddmmCSR{1,2}Scale (cogdl/operators/spmm/sddmm_kernel.cu:249-417) and mhsddmm
// (cogdl/operators/spmm/multiheadSddmm.cu:6-93).  Both reference kernels are edge-parallel and
// recover row(p) with a per-edge binary search over rowptr (computeUtil.h:36-53) and re-read
// the D1 row for every edge.  Here the work item is a row (or an edge chunk of a hub row):
// row(p) is free, the D1/grad row segment is loaded once into registers and only the D2/feat
// rows are gathered (4F bytes per edge instead of 8F).
//
// A dense row is seen as NSEG segments (heads) of L vectors each.  SUB lanes cooperate on one
// segment's dot product; a GROUP of lanes therefore covers GROUP/SUB segments at once
// (small F: all heads of an edge in one 512-byte gather), or one segment with NV vectors per
// lane (F >= 128).  Dot products are reduced with xor-shuffles inside the SUB lanes.
#include "common.cuh"

#include <cstdlib>

namespace cogdl_b200 {

struct SddmmParams {
  const int *rowptr;
  const int *colind;
  const float *D1;
  const float *D2;
  float *out;
  int64_t n_rows;
  int NSEG;   // segments (heads) per dense row
  int L;      // vectors per segment
  HubView hub;
};

__device__ __forceinline__ float vdot(const float4 &a, const float4 &b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ float vdot(const float &a, const float &b) { return a * b; }

// NV > 0: the lane keeps NV vectors of the D1 segment in registers (L <= SUB*NV).
// NV == 0: generic, loops over the segment (any L), re-reading D1 through L1.
template <typename VecT, int GROUP, int SUB, int NV>
__global__ void __launch_bounds__(256) sddmm_kernel(const SddmmParams p) {
  static_assert(SUB <= GROUP && GROUP <= 32, "bad shape");
  constexpr int SPG = GROUP / SUB;          // segments per group
  constexpr int NVR = NV > 0 ? NV : 1;
  constexpr int U0 = NV <= 1 ? 4 : 2;
  constexpr int U = U0 < GROUP ? U0 : GROUP;
  const int lane = threadIdx.x & 31;
  const int gl = lane & (GROUP - 1);
  const int sl = gl & (SUB - 1);            // lane inside the segment team
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const WorkItem w = decode_item(tid / GROUP, p.n_rows, p.rowptr, p.hub);

  const int seg = blockIdx.y * SPG + gl / SUB;
  const bool segok = seg < p.NSEG;
  const int64_t ld = (int64_t)p.NSEG * p.L;  // dense row length in vectors
  const VecT *D1 = reinterpret_cast<const VecT *>(p.D1);
  const VecT *D2 = reinterpret_cast<const VecT *>(p.D2);

  VecT a[NVR];
  bool colok[NVR];
#pragma unroll
  for (int k = 0; k < NVR; ++k) {
    colok[k] = segok && (sl + k * SUB) < p.L;
    if (NV > 0 && colok[k] && w.lb < w.hb) a[k] = __ldg(D1 + (int64_t)w.row * ld + (int64_t)seg * p.L + sl + k * SUB);
  }

  int maxdeg = w.hb - w.lb;
  if (GROUP < 32) maxdeg = warp_max(maxdeg);

  for (int off = 0; off < maxdeg; off += GROUP) {
    const int cnt = min(GROUP, w.hb - w.lb - off);
    int c = 0;
    if (gl < cnt) c = ld_stream(p.colind + w.lb + off + gl);
#pragma unroll 1
    for (int j = 0; j < GROUP; j += U) {
      if (GROUP == 32) {
        if (j >= cnt) break;
      } else {
        if (!__any_sync(FULL, j < cnt)) break;
      }
      float d[U];
      if (NV > 0) {
        VecT b[U][NVR];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, c, j + u, GROUP);
          if (j + u < cnt) {
            const VecT *bp = D2 + (int64_t)cj * ld + (int64_t)seg * p.L + sl;
#pragma unroll
            for (int k = 0; k < NVR; ++k)
              if (colok[k]) b[u][k] = ld_gather(bp + k * SUB);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          d[u] = 0.f;
          if (j + u < cnt) {
#pragma unroll
            for (int k = 0; k < NVR; ++k)
              if (colok[k]) d[u] += vdot(a[k], b[u][k]);
          }
        }
      } else {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cj = __shfl_sync(FULL, c, j + u, GROUP);
          d[u] = 0.f;
          if (j + u < cnt && segok) {
            const VecT *ap = D1 + (int64_t)w.row * ld + (int64_t)seg * p.L;
            const VecT *bp = D2 + (int64_t)cj * ld + (int64_t)seg * p.L;
            for (int t = sl; t < p.L; t += SUB) d[u] += vdot(__ldg(ap + t), ld_gather(bp + t));
          }
        }
      }
      // reduce the U dot products inside each SUB-lane team (interleaved butterflies)
#pragma unroll
      for (int s = SUB / 2; s > 0; s >>= 1) {
#pragma unroll
        for (int u = 0; u < U; ++u) d[u] += __shfl_xor_sync(FULL, d[u], s);
      }
      // team lane u writes edge j+u (SUB >= U) -- otherwise team lane 0 writes them all
      if (segok) {
        if (SUB >= U) {
#pragma unroll
          for (int u = 0; u < U; ++u)
            if (sl == u && j + u < cnt) p.out[(int64_t)(w.lb + off + j + u) * p.NSEG + seg] = d[u];
        } else if (sl == 0) {
#pragma unroll
          for (int u = 0; u < U; ++u)
            if (j + u < cnt) p.out[(int64_t)(w.lb + off + j + u) * p.NSEG + seg] = d[u];
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Row-stream form (plan with segments, F a multiple of 128 per head, float4 path): one warp per
// (edge range, head) where the edge ranges are the plan's hub chunks and segments.  Outputs are per
// edge, so chunks and segments are the same thing here: no flush, no partials.  Both operands are
// gathered per edge -- the left one (D1 / grad row of the edge's OWN row, via edge_row) repeats for
// consecutive edges of a row and is served by L1 -- so every batch has 2*U independent 512-byte
// loads in flight and there is no per-row reload latency.
// ------------------------------------------------------------------------------------------
template <int NV, int U>
__global__ void __launch_bounds__(256) sddmm_stream_kernel(const SddmmParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t item = wid / p.NSEG;
  const int head = (int)(wid - item * p.NSEG);
  int e, e_end, fixed_row = -1;
  if (item < p.hub.n_chunks) {
    const WorkItem w = decode_item(item, 0, p.rowptr, p.hub);
    e = w.lb; e_end = w.hb; fixed_row = w.row;
  } else {
    const int64_t seg = item - p.hub.n_chunks;
    if (seg >= p.hub.n_segs) return;
    const int2 rr = __ldg(p.hub.segs + seg);
    e = __ldg(p.rowptr + rr.x); e_end = __ldg(p.rowptr + rr.y);
  }
  const int64_t ld = (int64_t)p.NSEG * p.L;
  const float4 *D1 = reinterpret_cast<const float4 *>(p.D1) + (int64_t)head * p.L + lane;
  const float4 *D2 = reinterpret_cast<const float4 *>(p.D2) + (int64_t)head * p.L + lane;
  for (; e < e_end; e += 32) {
    const int cnt = min(32, e_end - e);
    int c = 0, r = 0;
    if (lane < cnt) {
      c = ld_stream(p.colind + e + lane);
      r = fixed_row >= 0 ? fixed_row : ld_stream(p.hub.edge_row + e + lane);
    }
#pragma unroll 1
    for (int j = 0; j < cnt; j += U) {
      float4 a[U][NV], b[U][NV];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int cj = __shfl_sync(FULL, c, j + u);
        const int rj = __shfl_sync(FULL, r, j + u);
        if (j + u < cnt) {
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            a[u][k] = __ldg(D1 + (int64_t)rj * ld + 32 * k);
            b[u][k] = ld_gather(D2 + (int64_t)cj * ld + 32 * k);
          }
        }
      }
      float d[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        d[u] = 0.f;
        if (j + u < cnt) {
#pragma unroll
          for (int k = 0; k < NV; ++k) d[u] += vdot(a[u][k], b[u][k]);
        }
      }
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
        for (int u = 0; u < U; ++u) d[u] += __shfl_xor_sync(FULL, d[u], s);
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (lane == u && j + u < cnt) p.out[(int64_t)(e + j + u) * p.NSEG + head] = d[u];
    }
  }
}

// Stream form vs row form, measured on an H100 SXM (700 W, arxiv shape, two alternating runs): 220 vs 298 us (F=128),
// 2.03 vs 2.53 ms (H=8, F=128) -> the stream form whenever the plan has segments and L is 32 or 64 vectors; the row
// form serves every other width and plans without segments.
template <int NV>
static int launch_sddmm_stream(const SddmmParams &p, cudaStream_t stream) {
  const int64_t warps = ((int64_t)p.hub.n_chunks + p.hub.n_segs) * p.NSEG;
  const int64_t blocks = ceil_div(warps * 32, 256);
  if (blocks == 0) return COGDL_B200_OK;
  if (blocks > 0x7fffffffLL) return set_error(COGDL_B200_EINVAL, "sddmm: problem too large for one launch");
  constexpr int U = NV == 1 ? 4 : 2;
  note_kernel("cogdl_b200::sddmm_stream_kernel<NV=%d,U=%d>", NV, U);
  sddmm_stream_kernel<NV, U><<<(unsigned)blocks, 256, 0, stream>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

template <typename VecT, int GROUP, int SUB, int NV>
static int launch_sddmm(const SddmmParams &p, cudaStream_t stream) {
  const int64_t items = (int64_t)p.hub.n_chunks + p.n_rows;
  const int64_t blocks = ceil_div(items * GROUP, 256);
  const int64_t ytiles = ceil_div(p.NSEG, GROUP / SUB);
  if (blocks == 0 || ytiles == 0) return COGDL_B200_OK;
  if (blocks > 0x7fffffffLL || ytiles > 65535)
    return set_error(COGDL_B200_EINVAL, "sddmm: problem too large for one launch");
  note_kernel("cogdl_b200::sddmm_kernel<%s,GROUP=%d,SUB=%d,NV=%d>", sizeof(VecT) == 16 ? "float4" : "float", GROUP, SUB, NV);
  sddmm_kernel<VecT, GROUP, SUB, NV><<<dim3((unsigned)blocks, (unsigned)ytiles), 256, 0, stream>>>(p);
  CB_LAUNCH_CHECK();
  return COGDL_B200_OK;
}

// Pick (GROUP, SUB, NV) for `NSEG` segments of `L` vectors.
template <typename VecT>
static int dispatch_sddmm(const SddmmParams &p, cudaStream_t s) {
  const int L = p.L, H = p.NSEG;
  if constexpr (sizeof(VecT) == 16) {
    if (p.hub.n_segs > 0) {
      if (L == 32) return launch_sddmm_stream<1>(p, s);
      if (L == 64) return launch_sddmm_stream<2>(p, s);
    }
  }
  if (L > 128) return launch_sddmm<VecT, 32, 32, 0>(p, s);
  if (L > 64) return launch_sddmm<VecT, 32, 32, 4>(p, s);
  if (L > 32) return launch_sddmm<VecT, 32, 32, 2>(p, s);
  if (L > 16) return launch_sddmm<VecT, 32, 32, 1>(p, s);
  // L <= 16: several segments per warp when there are several heads
  if (L > 8) return (H >= 2) ? launch_sddmm<VecT, 32, 16, 1>(p, s) : launch_sddmm<VecT, 16, 16, 1>(p, s);
  if (L > 4) {
    if (H >= 4) return launch_sddmm<VecT, 32, 8, 1>(p, s);
    if (H >= 2) return launch_sddmm<VecT, 16, 8, 1>(p, s);
    return launch_sddmm<VecT, 8, 8, 1>(p, s);
  }
  if (L > 2) {
    if (H >= 8) return launch_sddmm<VecT, 32, 4, 1>(p, s);
    if (H >= 4) return launch_sddmm<VecT, 16, 4, 1>(p, s);
    if (H >= 2) return launch_sddmm<VecT, 8, 4, 1>(p, s);
    return launch_sddmm<VecT, 4, 4, 1>(p, s);
  }
  if (L > 1) {
    if (H >= 8) return launch_sddmm<VecT, 16, 2, 1>(p, s);
    if (H >= 4) return launch_sddmm<VecT, 8, 2, 1>(p, s);
    return launch_sddmm<VecT, 4, 2, 1>(p, s);
  }
  if (H >= 8) return launch_sddmm<VecT, 8, 1, 1>(p, s);
  if (H >= 4) return launch_sddmm<VecT, 4, 1, 1>(p, s);
  if (H >= 2) return launch_sddmm<VecT, 2, 1, 1>(p, s);
  return launch_sddmm<VecT, 1, 1, 1>(p, s);
}

static int sddmm_entry(const int32_t *rowptr, const int32_t *colind, const float *D1, const float *D2,
                       float *out, int64_t n_rows, int64_t H, int64_t F,
                       const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream, const char *who) {
  CB_REQUIRE(n_rows >= 0 && H >= 0 && F >= 0, "%s: negative size", who);
  if (n_rows == 0 || H == 0) return COGDL_B200_OK;
  CB_REQUIRE(rowptr && colind && out, "%s: null pointer", who);
  CB_REQUIRE(F == 0 || (D1 && D2), "%s: null pointer", who);
  CB_REQUIRE(n_rows < 0x7fffffffLL && H * F < 0x7fffffffLL, "%s: sizes must fit int32", who);
  int rc = check_plan(plan, 0);
  if (rc) return rc;
  SddmmParams p;
  p.rowptr = rowptr; p.colind = colind; p.D1 = D1; p.D2 = D2; p.out = out; p.n_rows = n_rows;
  p.NSEG = (int)H; p.hub = hub_view(plan);
  if (F % 4 == 0 && aligned16(D1) && aligned16(D2)) {
    p.L = (int)(F / 4);
    return dispatch_sddmm<float4>(p, (cudaStream_t)stream);
  }
  p.L = (int)F;
  return dispatch_sddmm<float>(p, (cudaStream_t)stream);
}

}  // namespace cogdl_b200

using namespace cogdl_b200;

extern "C" int cogdl_b200_sddmm_csr_f32(const int32_t *rowptr, const int32_t *colind, const float *D1,
                                        const float *D2, float *out, int64_t n_rows, int64_t F,
                                        const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return sddmm_entry(rowptr, colind, D1, D2, out, n_rows, 1, F, plan, stream, "cogdl_b200_sddmm_csr_f32");
}

extern "C" int cogdl_b200_mhsddmm_f32(const int32_t *rowptr, const int32_t *colind, const float *grad,
                                      const float *feat, float *out, int64_t n_rows, int64_t H, int64_t F,
                                      const cogdl_b200_hub_plan_t *plan, cogdl_b200_stream_t stream) {
  return sddmm_entry(rowptr, colind, grad, feat, out, n_rows, H, F, plan, stream, "cogdl_b200_mhsddmm_f32");
}

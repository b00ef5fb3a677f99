// pwpp_kernels.cuh — the sm_90a kernels of the estimateGround() path.
//
//   k_bin_hist   RNR predicate + polar bin id per point + per-chunk bin histogram
//                (reference reflected_noise_removal S:377-400, pc2czm S:578-622, flush_patches S:33-45)
//   k_bin_scan   per frame: bin offsets + per-(chunk,bin) scatter bases  (replaces the emplace_back
//                growth of czm[k][i][j], S:602-614)
//   k_scatter    stable, deterministic scatter of (x,y,z,idx) into bin-contiguous order, ascending
//                point index inside a bin — the order pc2czm produces
//   k_fit        per bin: LPR seed selection, R-VPF, R-GPF plane fits, ground/non-ground split
//                (sort S:199 [not needed, see below], extract_piecewiseground S:467-549,
//                 extract_initial_seeds S:77-149, estimate_plane S:47-75, calc_point_to_plane_d S:551-554)
//   k_gle        per frame: A-GLE verdicts, TGR, adaptive threshold + sensor-height update, output
//                segment layout in the reference's emission order
//                (S:211-311, temporal_ground_revert S:402-464, update_* S:338-375)
//   k_emit       copies every bin's ground / non-ground part to the final index lists
//                (addCloud S:28-31 + toIndices S:18-26)
//   k_gather_xyz toEigenCloud S:8-16 on demand
//
// "S:" = reference cpp/patchworkpp/src/patchworkpp.cpp, "H:" = .../include/patchwork/patchworkpp.h.
#pragma once
#include <cuda_runtime.h>

#include "pwpp_common.cuh"
#include "pwpp_fit.cuh"
#include "pwpp_fit_big.cuh"
#include "pwpp_fit_patch.cuh"
#include "pwpp_order.cuh"
#include "pwpp_front.cuh"

namespace pwpp {

// ---------------------------------------------------------------------------------------------------
// k_bin_hist: grid (max_chunks_per_frame, F), 256 threads. Each warp owns 512 consecutive points.
// Writes bin ids (u16) and the chunk's histogram row (u16[nbp]).
// PIPE: 0 = load a group of 4 points per lane, bin them, repeat; 1 / 2 = groups of 4 / 2 with the next group's loads in
// flight while the current one is binned (PWPP_HIST_PIPE, A/B switch)
template <bool FAST, int PIPE>
__global__ void __launch_bounds__(CHUNK_THREADS, 4) k_bin_hist(const float4* __restrict__ pts, FrameTable ft, const StreamState* __restrict__ states,
                                                             const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps,
                                                             int has_intensity, int nbp,
                                                             unsigned short* __restrict__ bin_ids, unsigned short* __restrict__ chist) {
  PW_DYN_SHARED(unsigned int, s_hist);  // [nbp]
  const int f = blockIdx.y;
  const long long p0 = ft.pt_off[f];
  const int n = (int) (ft.pt_off[f + 1] - p0);
  const int nchunks = (n + CHUNK_PTS - 1) / CHUNK_PTS;
  if ((int) blockIdx.x >= nchunks) return;
  for (int b = threadIdx.x; b < nbp; b += CHUNK_THREADS) s_hist[b] = 0;
  __syncthreads();
  const int set = ft.pset[f];   // the frame's parameter set
  const Geometry& g = gs.g[set];
  const AlgoParams& ap = aps.a[set];
  const double sensor_height = states[ft.stream[f]].sensor_height;
  const bool rnr_on = ap.enable_RNR && has_intensity;  // S:161, S:379-382
  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int base = blockIdx.x * CHUNK_PTS + warp * WARP_PTS;
  constexpr int HB = PIPE == 2 ? 2 : 4;   // points per load group and lane
  const int last = n - 1;
  float4 q[HB], qn[HB];
#pragma unroll
  for (int u = 0; u < HB; ++u) { const int i = base + u * 32 + lane; q[u] = ld_stream_f4(pts + p0 + (i < n ? i : last)); }
#pragma unroll 1
  for (int h = 0; h < WARP_ITERS; h += HB) {
    if (PIPE != 0 && h + HB < WARP_ITERS) {
#pragma unroll
      for (int u = 0; u < HB; ++u) { const int i = base + (h + HB + u) * 32 + lane; qn[u] = ld_stream_f4(pts + p0 + (i < n ? i : last)); }
    }
#pragma unroll
    for (int u = 0; u < HB; ++u) {
      const int i = base + (h + u) * 32 + lane;
      const float4 p = q[u];
      int bin = -1;
      if (i < n) {
        if (rnr_on && rnr_hit(p.x, p.y, p.z, p.w, sensor_height, ap)) bin = PW_BIN_RNR(g.nbins);
        else if (p.z == FLT_MIN) bin = PW_BIN_DROP(g.nbins);  // S:591
        else bin = FAST ? bin_of_point(p.x, p.y, p.z, g) : bin_of_point_exact(p.x, p.y, p.z, g);
        bin_ids[p0 + i] = (unsigned short) bin;
      }
      // warp-aggregated histogram update: one shared atomic per distinct bin in the warp
      const unsigned act = __ballot_sync(0xffffffffu, bin >= 0);
      if (bin >= 0) {
        const unsigned peers = __match_any_sync(act, bin);
        if ((peers & lanemask_lt()) == 0) atomicAdd(&s_hist[bin], __popc(peers));
      }
    }
    if (PIPE != 0) {
#pragma unroll
      for (int u = 0; u < HB; ++u) q[u] = qn[u];
    } else if (h + HB < WARP_ITERS) {
#pragma unroll
      for (int u = 0; u < HB; ++u) { const int i = base + (h + HB + u) * 32 + lane; q[u] = ld_stream_f4(pts + p0 + (i < n ? i : last)); }
    }
  }
  __syncthreads();
  unsigned short* row = chist + (size_t) (ft.chunk_off[f] + blockIdx.x) * nbp;
  for (int b = threadIdx.x; b < nbp; b += CHUNK_THREADS) row[b] = (unsigned short) s_hist[b];
}

// ---------------------------------------------------------------------------------------------------
// k_bin_scan: one CTA per frame, thread b <-> bin b (striding when nbp > blockDim.x).
// bin_off[f][b] = first position of bin b inside the frame's sorted region ([nbp+1] entries);
// cbase[chunk][b] = position where chunk's first point of bin b goes.
// Also sorts the frame's patches into the work queues of the fit kernels by size (S:191: patches below
// num_min_pts are not fitted) and initialises the BinFit records of the patches that will not be fitted.
// nbs is the stride of the patch records; the frame's bin count and num_min_pts are those of its parameter set.
template <int L2MAX, int MMAX = CLS_M_MAX>
__global__ void k_bin_scan(FrameTable ft, int nbp, int nbs, const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps,
                           const unsigned short* __restrict__ chist, unsigned int* __restrict__ cbase, int* __restrict__ bin_off, WorkQueues wq,
                           BinFit* __restrict__ fits) {
  PW_DYN_SHARED(int, s_scan);  // [nbp + 1]
  __shared__ int s_cls_cnt[NUM_CLASSES], s_cls_base[NUM_CLASSES], s_cls_pos[NUM_CLASSES];
  const int f = blockIdx.x;
  const int set = ft.pset[f];
  const int nbins = gs.g[set].nbins, num_min_pts = aps.a[set].num_min_pts;
  const int c0 = ft.chunk_off[f], c1 = ft.chunk_off[f + 1];
  if (threadIdx.x < NUM_CLASSES) { s_cls_cnt[threadIdx.x] = 0; s_cls_pos[threadIdx.x] = 0; }
  for (int b = threadIdx.x; b < nbp; b += blockDim.x) {
    int tot = 0;
    for (int c = c0; c < c1; ++c) tot += chist[(size_t) c * nbp + b];
    s_scan[b] = tot;
  }
  __syncthreads();
  // exclusive scan over nbp (<= 4096) values by warp 0: simple and tiny
  if (threadIdx.x < 32) {
    int carry = 0;
    for (int b0 = 0; b0 < nbp; b0 += 32) {
      const int b = b0 + threadIdx.x;
      int v = b < nbp ? s_scan[b] : 0;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if ((int) threadIdx.x >= o) incl += t; }
      if (b < nbp) s_scan[b] = carry + incl - v;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (threadIdx.x == 0) s_scan[nbp] = carry;
  }
  __syncthreads();
  int* bo = bin_off + (size_t) f * (nbp + 1);
  for (int b = threadIdx.x; b <= nbp; b += blockDim.x) bo[b] = s_scan[b];
  for (int b = threadIdx.x; b < nbp; b += blockDim.x) {
    unsigned int run = (unsigned int) s_scan[b];
    for (int c = c0; c < c1; ++c) {
      const unsigned int v = chist[(size_t) c * nbp + b];
      cbase[(size_t) c * nbp + b] = run;
      run += v;
    }
  }
  // work queues
  auto cls_of = [](int n) { return n <= CLS_S_MAX ? 0 : n <= MMAX ? 1 : n <= CLS_L1_MAX ? 2 : n <= L2MAX ? 3 : n <= CLS_L3_MAX ? 4 : 5; };
  for (int b = threadIdx.x; b < nbins; b += blockDim.x) {
    const int n = s_scan[b + 1] - s_scan[b];
    if (n >= num_min_pts && n > 0) atomicAdd(&s_cls_cnt[cls_of(n)], 1);
    else {
      BinFit& r = fits[(size_t) f * nbs + b];
      r.n = n; r.n_ground = 0; r.d = 0.0;
      for (int k = 0; k < 3; ++k) { r.mean[k] = 0.0; r.normal[k] = 0.0; r.sv[k] = 0.0; }
      // an EMPTY patch with num_min_pts <= 0 is "fitted" by the reference with the previous patch's plane (S:49)
      r.fitted = (n >= num_min_pts) ? 1 : 0;
      r.verdict = r.fitted ? PW_FIT_NO_PLANE : 0;
    }
  }
  __syncthreads();
  if (threadIdx.x < NUM_CLASSES) s_cls_base[threadIdx.x] = s_cls_cnt[threadIdx.x] ? atomicAdd(&wq.count[threadIdx.x], s_cls_cnt[threadIdx.x]) : 0;
  __syncthreads();
  for (int b = threadIdx.x; b < nbins; b += blockDim.x) {
    const int n = s_scan[b + 1] - s_scan[b];
    if (n >= num_min_pts && n > 0) {
      const int c = cls_of(n);
      wq.items[c][s_cls_base[c] + atomicAdd(&s_cls_pos[c], 1)] = make_work_item(f, b, n, ft.pt_off[f] + (long long) s_scan[b]);
    }
  }
}

#if defined(PWPP_SIMT_EMU)
// tests/simt: the one-set launch with the frame's bin count and num_min_pts as scalars (what the CPU twin passes)
template <int L2MAX, int MMAX = CLS_M_MAX>
inline void k_bin_scan(FrameTable ft, int nbp, int nbins, int num_min_pts, const unsigned short* chist, unsigned int* cbase, int* bin_off, WorkQueues wq,
                       BinFit* fits) {
  Geometry g{};
  g.nbins = nbins;
  AlgoParams ap{};
  ap.num_min_pts = num_min_pts;
  k_bin_scan<L2MAX, MMAX>(ft, nbp, nbins, GeometrySets(g), AlgoParamSets(ap), chist, cbase, bin_off, wq, fits);
}
#endif

// ---------------------------------------------------------------------------------------------------
// k_scatter: same decomposition as k_bin_hist. Stable: a point's position inside its bin is its rank
// among the frame's points of that bin in ascending point index.
//   rank = cbase[chunk][bin] + (#points of bin in lower warps of the chunk)
//        + (#points of bin in earlier iterations of this warp) + (#lower lanes with the same bin)
// The kernel is latency-bound (few active warps, mostly long-scoreboard stalls, DRAM far from saturated), so what pays is
// resident warps: it is sized for 4 CTAs per SM (64 registers), which ran faster than 2 CTAs per SM. PIPE = true additionally software-pipelines the point loads in two groups of SB, the first two issued
// before the histogram / prefix phases; measured equal at 3 CTAs per SM, kept as the PWPP_SCATTER_V=1 variant.
template <bool PIPE, int MINB>
__global__ void __launch_bounds__(CHUNK_THREADS, MINB) k_scatter(const float4* __restrict__ pts, FrameTable ft, int nbp,
                                                               const unsigned short* __restrict__ bin_ids, const unsigned int* __restrict__ cbase,
                                                               float4* __restrict__ sorted) {
  PW_DYN_SHARED(unsigned int, s_wcnt);  // [8][nbp]: per-warp histograms, then per-warp running positions
  const int f = blockIdx.y;
  const long long p0 = ft.pt_off[f];
  const int n = (int) (ft.pt_off[f + 1] - p0);
  const int nchunks = (n + CHUNK_PTS - 1) / CHUNK_PTS;
  if ((int) blockIdx.x >= nchunks) return;
  const int nwarps = CHUNK_THREADS / 32;
  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int base = blockIdx.x * CHUNK_PTS + warp * WARP_PTS;
  const int last = n - 1;
  constexpr int SB = 4;   // points per load group and lane
  float4 qa[SB], qb[SB];
  auto load_group = [&](float4 (&q)[SB], int h) {
#pragma unroll
    for (int u = 0; u < SB; ++u) { const int i = base + (h + u) * 32 + lane; q[u] = ld_stream_f4(pts + p0 + (i < n ? i : last)); }
  };
  if (PIPE) { load_group(qa, 0); load_group(qb, SB); }
  for (int b = threadIdx.x; b < nwarps * nbp; b += CHUNK_THREADS) s_wcnt[b] = 0;
  __syncthreads();
  unsigned int* my = s_wcnt + warp * nbp;
  int bins[WARP_ITERS];
  // all 16 bin ids of the lane are requested before the first one is used (__syncwarp below is a memory barrier the
  // compiler will not move loads across)
#pragma unroll
  for (int it = 0; it < WARP_ITERS; ++it) {
    const int i = base + it * 32 + lane;
    bins[it] = (i < n) ? (int) bin_ids[p0 + i] : -1;
  }
#pragma unroll
  for (int it = 0; it < WARP_ITERS; ++it) {
    const int bin = bins[it];
    const unsigned act = __ballot_sync(0xffffffffu, bin >= 0);
    if (bin >= 0) {
      const unsigned peers = __match_any_sync(act, bin);
      if ((peers & lanemask_lt()) == 0) my[bin] += __popc(peers);  // only this warp writes its row
    }
    __syncwarp();
  }
  __syncthreads();
  // per bin: exclusive prefix over the 8 warps, offset by the chunk's base
  const unsigned int* cb = cbase + (size_t) (ft.chunk_off[f] + blockIdx.x) * nbp;
  for (int b = threadIdx.x; b < nbp; b += CHUNK_THREADS) {
    unsigned int run = cb[b];
#pragma unroll
    for (int w = 0; w < nwarps; ++w) { const unsigned int v = s_wcnt[w * nbp + b]; s_wcnt[w * nbp + b] = run; run += v; }
  }
  __syncthreads();
  float4* out = sorted + p0;
  auto place_group = [&](const float4 (&q)[SB], int h) {
#pragma unroll
    for (int u = 0; u < SB; ++u) {
      const int i = base + (h + u) * 32 + lane;
      const int bin = bins[h + u];
      const unsigned act = __ballot_sync(0xffffffffu, bin >= 0);
      if (bin >= 0) {
        const unsigned peers = __match_any_sync(act, bin);
        const unsigned int pos = my[bin] + __popc(peers & lanemask_lt());
        float4 p = q[u];
        p.w = __int_as_float(i);
        out[pos] = p;
        __syncwarp(peers);
        if ((peers & lanemask_lt()) == 0) my[bin] += __popc(peers);
      }
      __syncwarp();
    }
  };
  static_assert(WARP_ITERS % (2 * SB) == 0, "two load groups per pipeline step");
  if (PIPE) {
#pragma unroll
    for (int h = 0; h < WARP_ITERS; h += 2 * SB) {
      place_group(qa, h);
      if (h + 2 * SB < WARP_ITERS) load_group(qa, h + 2 * SB);
      place_group(qb, h + SB);
      if (h + 3 * SB < WARP_ITERS) load_group(qb, h + 3 * SB);
    }
  } else {
#pragma unroll
    for (int h = 0; h < WARP_ITERS; h += SB) {
      load_group(qa, h);
      place_group(qa, h);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// k_gle: one warp per frame. Same decisions as gle_frame()/update_thresholds() in tests/gle_sequential.cuh (the sequential
// statement of S:211-311, S:402-464, S:338-375 that the CPU twin runs) but lane-parallel over the sectors of a ring:
// per-sector flags are computed by the lanes, sequence-dependent quantities (history append positions, candidate
// order, output offsets) come from ballots / warp scans, and the per-array sums of calc_mean_stdev stay sequential
// inside one lane so that thresholds are bit-identical to the sequential code.
__device__ __forceinline__ int warp_excl_scan(int v, int& total) {
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane_id() >= o) incl += t; }
  total = __shfl_sync(0xffffffffu, incl, 31);
  return incl - v;
}
constexpr int GLE_CH = 128;   // samples of each history row staged per step of the threshold update
__host__ __device__ inline size_t gle_smem_bytes(int max_sectors) { return (size_t) 6 * max_sectors * sizeof(double) + (size_t) 2 * max_sectors * sizeof(int) + (size_t) 8 * GLE_CH * sizeof(double); }
#define PW_SEG_TO_NG(x) (-3 - (x))   /* "ground part goes to the non-ground list at offset x" until the final shift */

// hist_stride is the row stride of the histories (the largest history_cap of the sets); the logical capacity of a stream's rows
// is its own set's history_cap, exactly as in a context created with that set alone. max_sectors sizes the shared memory.
__global__ void __launch_bounds__(32) k_gle(FrameTable ft, StreamState* __restrict__ states, double* __restrict__ hist, int hist_stride,
                                            const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps, int nbp, int max_sectors, const int* __restrict__ bin_off, BinFit* __restrict__ fits, BinSeg* __restrict__ segs,
                                            int* __restrict__ num_ground, int* __restrict__ num_patches, float* __restrict__ centers, float* __restrict__ normals,
                                            int* __restrict__ num_dropped) {
  PW_DYN_SHARED(double, s_gle);
  double* s_rf = s_gle;                               // ringwise_flatness (S:182): [4 * max_sectors]
  double* s_clv = s_rf + 4 * max_sectors;             // candidates of the ring: line_variable [max_sectors]
  double* s_cfl = s_clv + max_sectors;                //                         flatness      [max_sectors]
  int* s_cbin = reinterpret_cast<int*>(s_cfl + max_sectors);  //                 bin           [max_sectors]
  int* s_cng = s_cbin + max_sectors;                  //                         |ground part| [max_sectors]
  const int rf_cap = 4 * max_sectors;
  const int f = blockIdx.x;
  const int lane = lane_id();
  const unsigned lt = lanemask_lt();
  const int sid = ft.stream[f];                       // frame f of the call advances stream sid
  const int set = ft.pset[f];                         // with the parameters of its set
  const Geometry& g = gs.g[set];
  const AlgoParams& ap = aps.a[set];
  StreamState& st = states[sid];
  const int nb = g.nbins, nb_all = nb + PW_NUM_PSEUDO;
  const int hcap = history_cap(g, ap);
  const int* bo = bin_off + (size_t) f * (nbp + 1);
  BinFit* fit = fits + (size_t) f * gs.nbs;
  BinSeg* seg = segs + (size_t) f * (gs.nbs + PW_NUM_PSEUDO);
  float* cen = centers + (size_t) f * gs.nbs * 3;
  float* nor = normals + (size_t) f * gs.nbs * 3;
  double* h_elev = hist + ((size_t) sid * 2 + 0) * 4 * hist_stride;
  double* h_flat = hist + ((size_t) sid * 2 + 1) * 4 * hist_stride;

#if !defined(PWPP_SIMT_EMU)
  // The ring loop below is a chain of ~20 dependent round trips to this frame's patch records (104 B each, written by the fit
  // kernels: L2 hits); one frame per call — the reference's pattern — has nothing else to hide them behind. Pull the
  // records (52 KB for the default 504 bins) into this SM's L1 up front: the loop then runs at L1 latency.
  {
    const char* base = reinterpret_cast<const char*>(fit);
    const int bytes = nb * (int) sizeof(BinFit);
    if (bytes <= 96 * 1024)
      for (int o = lane * 128; o < bytes; o += 32 * 128) asm volatile("prefetch.global.L1 [%0];" ::"l"(base + o));
  }
#endif
  const int n_rnr = bo[PW_BIN_RNR(nb) + 1] - bo[PW_BIN_RNR(nb)];
  const int n_oor = bo[PW_BIN_OOR(nb) + 1] - bo[PW_BIN_OOR(nb)];
  const int n_drop = bo[PW_BIN_DROP(nb) + 1] - bo[PW_BIN_DROP(nb)];
  if (lane == 0) {
    seg[PW_BIN_RNR(nb)].g_dst = -1; seg[PW_BIN_RNR(nb)].ng_dst = 0;
    seg[PW_BIN_OOR(nb)].g_dst = -1; seg[PW_BIN_OOR(nb)].ng_dst = n_rnr;
    seg[PW_BIN_DROP(nb)].g_dst = -1; seg[PW_BIN_DROP(nb)].ng_dst = -1;
  }
  int g_run = 0, ng_run = n_rnr + n_oor;
  int concentric = 0, npatch = 0, n_rf = 0;
  int n_e[4], n_f[4];
  double thr_e[4], thr_f[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { n_e[i] = st.n_elev[i]; n_f[i] = st.n_flat[i]; thr_e[i] = st.elevation_thr[i]; thr_f[i] = st.flatness_thr[i]; }
  double carry[9];
#pragma unroll
  for (int k = 0; k < 3; ++k) { carry[k] = st.stale_mean[k]; carry[3 + k] = st.stale_normal[k]; carry[6 + k] = st.stale_sv[k]; }

  for (int zone = 0; zone < 4; ++zone) {
    const int nsec = g.num_sectors[zone];
    for (int ring = 0; ring < g.num_rings[zone]; ++ring) {
      const bool near = concentric < ap.num_rings_of_interest;
      const int ci = near ? concentric : 0;
      int ncand = 0;
      for (int s0 = 0; s0 < nsec; s0 += 32) {
        const int sct = s0 + lane;
        const bool act = sct < nsec;
        const int b = g.bin_base[zone] + ring * nsec + (act ? sct : 0);
        double v[9];  // mean[0..2], normal[0..2], sv[0..2]
        int n = 0, n_gr = 0, fitted_i = 0, verdict_in = 0;
#pragma unroll
        for (int k = 0; k < 9; ++k) v[k] = 0.0;
        if (act) {
          const BinFit& r = fit[b];
          n = r.n; n_gr = r.n_ground; fitted_i = r.fitted; verdict_in = r.verdict;
          if (fitted_i && verdict_in != PW_FIT_NO_PLANE) {
#pragma unroll
            for (int k = 0; k < 3; ++k) { v[k] = r.mean[k]; v[3 + k] = r.normal[k]; v[6 + k] = r.sv[k]; }
          }
        }
        const bool fitted = act && fitted_i != 0;
        const bool no_plane = fitted && verdict_in == PW_FIT_NO_PLANE;
        const unsigned hp = __ballot_sync(0xffffffffu, fitted && !no_plane);
        const unsigned npm = __ballot_sync(0xffffffffu, no_plane);
        if (npm) {  // S:49: estimate_plane never ran on a non-empty set; the members keep the last plane in loop order
          const unsigned lower = hp & lt;
          const int src = lower ? (31 - __clz(lower)) : -1;
#pragma unroll
          for (int k = 0; k < 9; ++k) {
            const double t = __shfl_sync(0xffffffffu, v[k], src < 0 ? 0 : src);
            if (no_plane) v[k] = (src >= 0) ? t : carry[k];
          }
          if (no_plane) {
            BinFit& r = fit[b];
#pragma unroll
            for (int k = 0; k < 3; ++k) { r.mean[k] = v[k]; r.normal[k] = v[3 + k]; r.sv[k] = v[6 + k]; }
          }
        }
        const unsigned fm = __ballot_sync(0xffffffffu, fitted);
        if (fm) {
          const int last = 31 - __clz(fm);
#pragma unroll
          for (int k = 0; k < 9; ++k) carry[k] = __shfl_sync(0xffffffffu, v[k], last);
        }
        // S:211-212 centers / normals of every fitted patch, in loop order
        if (fitted) {
          const int pi = npatch + __popc(fm & lt);
#pragma unroll
          for (int k = 0; k < 3; ++k) { cen[pi * 3 + k] = (float) v[k]; nor[pi * 3 + k] = (float) v[3 + k]; }
        }
        npatch += __popc(fm);
        // S:217-246
        const double ground_uprightness = v[5], ground_elevation = v[2];
        double ground_flatness = v[6];
        if (v[7] < ground_flatness) ground_flatness = v[7];
        if (v[8] < ground_flatness) ground_flatness = v[8];
        const double line_variable = v[7] != 0 ? ddiv(v[6], v[7]) : DBL_MAX;
        double heading = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) heading = dadd(heading, dmul(v[k], v[3 + k]));
        const bool is_upright = ground_uprightness > ap.uprightness_thr;
        const bool is_heading_outside = heading < 0.0;
        bool is_not_elevated = false, is_flat = false;
        if (near) { is_not_elevated = ground_elevation < thr_e[ci]; is_flat = ground_flatness < thr_f[ci]; }
        // S:253-259 statistics, appended in sector order
        const bool push = fitted && is_upright && is_not_elevated && near;
        const unsigned pm = __ballot_sync(0xffffffffu, push);
        if (pm) {
          const int cnt = __popc(pm);
          double* he = h_elev + ci * hist_stride;
          double* hf = h_flat + ci * hist_stride;
          int ne = n_e[0], nf = n_f[0];
#pragma unroll
          for (int i = 1; i < 4; ++i) if (ci == i) { ne = n_e[i]; nf = n_f[i]; }
          if (ne + cnt <= hcap && nf + cnt <= hcap) {
            if (push) { const int r = __popc(pm & lt); he[ne + r] = ground_elevation; hf[nf + r] = ground_flatness; }
            ne += cnt; nf += cnt;
          } else {  // row full: sequential drop-oldest path (pwpp_gle.cuh history_push)
            for (unsigned m = pm; m; m &= m - 1) {
              const int l = __ffs(m) - 1;
              const double e = __shfl_sync(0xffffffffu, ground_elevation, l), fl = __shfl_sync(0xffffffffu, ground_flatness, l);
              if (lane == 0) { history_push(he, ne, hcap, e); history_push(hf, nf, hcap, fl); }
              ne = __shfl_sync(0xffffffffu, ne, 0); nf = __shfl_sync(0xffffffffu, nf, 0);
              __syncwarp();
            }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) if (ci == i) { n_e[i] = ne; n_f[i] = nf; }
          if (push) { const int r = n_rf + __popc(pm & lt); if (r < rf_cap) s_rf[r] = ground_flatness; }
          n_rf = (n_rf + cnt < rf_cap) ? n_rf + cnt : rf_cap;
        }
        // S:262-284 decision chain
        int verdict = 0;
        bool to_g = false, cand = false, rejected = false;
        if (fitted) {
          if (!is_upright) { verdict = 1; rejected = true; }
          else if (!near) { verdict = 2; to_g = true; }
          else if (!is_heading_outside) { verdict = 3; rejected = true; }
          else if (is_not_elevated || is_flat) { verdict = 4; to_g = true; }
          else { verdict = 6; cand = true; }
        }
        const unsigned cm = __ballot_sync(0xffffffffu, cand);
        if (cand) {
          const int r = ncand + __popc(cm & lt);
          s_cbin[r] = b; s_clv[r] = line_variable; s_cfl[r] = ground_flatness; s_cng[r] = n_gr;
        }
        ncand += __popc(cm);
        if (!fitted) n_gr = 0;
        const int ng_sz = act ? ((rejected ? n_gr : 0) + (n - n_gr)) : 0;
        const int g_sz = (act && to_g) ? n_gr : 0;
        int tot_ng, tot_g;
        const int ex_ng = warp_excl_scan(ng_sz, tot_ng);
        const int ex_g = warp_excl_scan(g_sz, tot_g);
        if (act) {
          BinSeg sg;
          if (rejected) { sg.g_dst = PW_SEG_TO_NG(ng_run + ex_ng); sg.ng_dst = ng_run + ex_ng + n_gr; }
          else { sg.ng_dst = ng_run + ex_ng; sg.g_dst = to_g ? (g_run + ex_g) : (cand ? -2 : -1); }
          seg[b] = sg;
          fit[b].verdict = verdict;
        }
        ng_run += tot_ng;
        g_run += tot_g;
      }
      if (ncand > 0) {  // S:292-304 (uniform branch)
        __syncwarp();
        double mean_flatness = 0.0, stdev_flatness = 0.0;
        if (ap.enable_TGR) calc_mean_stdev(s_rf, n_rf, mean_flatness, stdev_flatness);  // S:407-408, every lane redundantly
        for (int c0 = 0; c0 < ncand; c0 += 32) {
          const int c = c0 + lane;
          const bool act = c < ncand;
          bool revert = false;
          int cb = 0, cng = 0;
          if (act) {
            cb = s_cbin[c]; cng = s_cng[c];
            if (ap.enable_TGR) {  // temporal_ground_revert S:416-461
              const double flat = s_cfl[c];
              const double mu_flatness = dadd(mean_flatness, dmul(1.5, stdev_flatness));
              double prob_flatness = ddiv(1.0, dadd(1.0, exp(ddiv(dsub(flat, mu_flatness), ddiv(mu_flatness, 10.0)))));
              if (cng > 1500 && flat < dmul(ap.th_dist, ap.th_dist)) prob_flatness = 1.0;
              double prob_line = 1.0;
              if (s_clv[c] > 8.0) prob_line = 0.0;
              revert = dmul(prob_line, prob_flatness) > 0.5;
            }
          }
          int tot_g, tot_n;
          const int ex_g = warp_excl_scan((act && revert) ? cng : 0, tot_g);
          const int ex_n = warp_excl_scan((act && !revert) ? cng : 0, tot_n);
          if (act) {
            seg[cb].g_dst = revert ? (g_run + ex_g) : PW_SEG_TO_NG(ng_run + ex_n);
            fit[cb].verdict = revert ? 5 : 6;
          }
          g_run += tot_g;
          ng_run += tot_n;
        }
        n_rf = 0;
        __syncwarp();
      }
      concentric++;
    }
  }
  __syncwarp();
  // the non-ground list sits behind the ground list; decode the "ground part -> non-ground list" markers
  for (int b = lane; b < nb_all; b += 32) {
    BinSeg sg = seg[b];
    if (sg.ng_dst >= 0) sg.ng_dst += g_run;
    if (sg.g_dst <= -3) sg.g_dst = (-3 - sg.g_dst) + g_run;
    seg[b] = sg;
  }
  if (lane == 0) {
    num_ground[f] = g_run; num_patches[f] = npatch; num_dropped[f] = n_drop;
#pragma unroll
    for (int i = 0; i < 4; ++i) { st.n_elev[i] = n_e[i]; st.n_flat[i] = n_f[i]; }
#pragma unroll
    for (int k = 0; k < 3; ++k) { st.stale_mean[k] = carry[k]; st.stale_normal[k] = carry[3 + k]; st.stale_sv[k] = carry[6 + k]; }
  }
  __syncwarp();
  // update_elevation_thr S:338-357 / update_flatness_thr S:359-375: lane r (0..3) owns elevation ring r, lane 4+r
  // flatness ring r; each history is summed sequentially by its lane (same order as S:561-565).
  const int nroi = ap.num_rings_of_interest;
  double m = 0.0, sd = 0.0;
  int cnt = 0;
  bool elev_active = false;
  if (lane < 4) {
    if (lane < nroi) { cnt = n_e[0]; for (int i = 1; i < 4; ++i) if (lane == i) cnt = n_e[i]; elev_active = cnt > 0; }
  } else if (lane < 8) {
    const int r = lane - 4;
    if (r < nroi) { cnt = n_f[0]; for (int i = 1; i < 4; ++i) if (r == i) cnt = n_f[i]; }
  }
  {
    // calc_mean_stdev (S:557-566) of the eight histories at once: the whole warp stages GLE_CH samples of every row in
    // shared memory (coalesced loads), then lane r sums row r's samples in order — the same operations in the same order as
    // the sequential function, without a global-memory round trip per sample (a full history holds max_*_storage = 1000)
    double* s_h = reinterpret_cast<double*>(s_cng + max_sectors);   // [8][GLE_CH] (8-byte aligned: 2 * max_sectors ints precede it)
    const int my_n = (lane < 8 && cnt > 1) ? cnt : 0;               // calc_mean_stdev leaves mean / stdev untouched when n <= 1
    const int max_n = __reduce_max_sync(0xffffffffu, my_n);
    for (int pass = 0; pass < 2; ++pass) {
      double acc = 0.0;
      for (int c0 = 0; c0 < max_n; c0 += GLE_CH) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int nr = __shfl_sync(0xffffffffu, my_n, r);
          const double* src = (r < 4 ? h_elev + r * hist_stride : h_flat + (r - 4) * hist_stride) + c0;
          const int len = min(GLE_CH, nr - c0);
          for (int i = lane; i < len; i += 32) s_h[r * GLE_CH + i] = src[i];
        }
        __syncwarp();
        if (lane < 8) {
          const int len = min(GLE_CH, my_n - c0);
          const double* v = s_h + lane * GLE_CH;
          if (pass == 0) { for (int i = 0; i < len; ++i) acc = dadd(acc, v[i]); }
          else { for (int i = 0; i < len; ++i) { const double d = dsub(v[i], m); acc = dadd(acc, dmul(d, d)); } }
        }
        __syncwarp();
      }
      if (my_n > 1) {
        if (pass == 0) m = ddiv(acc, (double) my_n);
        else sd = dsqrt(ddiv(acc, (double) (my_n - 1)));
      }
    }
  }
  // the flatness loop BREAKS at the first ring with <= 1 samples (S:363-364)
  const unsigned flat_ok = __ballot_sync(0xffffffffu, lane >= 4 && lane < 8 && (lane - 4) < nroi && cnt > 1) >> 4;
  if (lane < 4 && elev_active) {
    if (lane == 0) { st.elevation_thr[0] = dadd(m, dmul(3.0, sd)); st.sensor_height = -m; }  // S:346-349
    else st.elevation_thr[lane] = dadd(m, dmul(2.0, sd));                                     // S:350
  }
  bool flat_upd = false;
  if (lane >= 4 && lane < 8 && (lane - 4) < nroi) {
    const int r = lane - 4;
    const unsigned need = (1u << (r + 1)) - 1u;
    flat_upd = (flat_ok & need) == need;
    if (flat_upd) st.flatness_thr[r] = dadd(m, sd);  // S:368
  }
  const unsigned flat_upd_mask = __ballot_sync(0xffffffffu, flat_upd) >> 4;
  __syncwarp();
  // keep the newest max_*_storage samples (S:354-355, S:372-373; the flatness erase sits behind the break)
  for (int r = 0; r < 4 && r < nroi; ++r) {
    for (int which = 0; which < 2; ++which) {
      int nn = which ? n_f[0] : n_e[0];
      for (int i = 1; i < 4; ++i) if (r == i) nn = which ? n_f[i] : n_e[i];
      const int exceed = nn - (which ? ap.max_flatness_storage : ap.max_elevation_storage);
      const bool doit = which ? (((flat_upd_mask >> r) & 1u) != 0) : (nn > 0);
      if (doit && exceed > 0) {
        double* a = (which ? h_flat : h_elev) + r * hist_stride;
        for (int i0 = 0; i0 < nn - exceed; i0 += 32) {
          const int i = i0 + lane;
          double t = 0.0;
          if (i < nn - exceed) t = a[i + exceed];
          __syncwarp();
          if (i < nn - exceed) a[i] = t;
          __syncwarp();
        }
        if (lane == 0) { if (which) st.n_flat[r] = nn - exceed; else st.n_elev[r] = nn - exceed; }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// k_emit: copies every patch's ground / non-ground part to its place in the final index lists (addCloud S:28-31 + toIndices
// S:18-26). Fitted patches were partitioned by the fit kernels (part[]: ground part, then non-ground part); patches that were not
// fitted (below num_min_pts, RNR hits, out-of-range points) are emitted straight from the sorted array in ascending point index.
// The ground part and the non-ground part of a bin are contiguous both in `part` / `sorted` and in the output lists.
// The work is cut by POSITION, not by bin: every warp owns EMIT_TILE consecutive positions of a
// frame's bin-sorted order, finds the bin of its first position (32-ary search over the bin offsets: two round trips for 507 bins),
// then walks the bins 32 at a time — offsets, destinations and ground counts of a window are loaded lane-parallel and broadcast by
// shuffles — and copies the intersection of every bin with its tile, four loads in flight per lane. All warps do the same amount of
// copying whatever the bin sizes are. It replaced a slower first form, one warp per bin (most warps owned a tiny bin and spent their
// time in the three dependent loads before the copy loop; the 20k..40k-point bins of a dense frame had to be split over 16 warps).
constexpr int EMIT_WARPS = 8;
constexpr int EMIT_TILE = 1024;

__global__ void __launch_bounds__(EMIT_WARPS * 32) k_emit(FrameTable ft, const __grid_constant__ GeometrySets gs, int nbp, const int* __restrict__ bin_off, const BinFit* __restrict__ fits,
                                                                const BinSeg* __restrict__ segs, const int* __restrict__ part, const float4* __restrict__ sorted,
                                                                int* __restrict__ out_idx) {
  const int f = blockIdx.y;
  const int lane = lane_id();
  const long long p0 = ft.pt_off[f];
  const int n = (int) (ft.pt_off[f + 1] - p0);
  const int w0 = (blockIdx.x * EMIT_WARPS + (threadIdx.x >> 5)) * EMIT_TILE;
  if (w0 >= n) return;
  const int w1 = min(n, w0 + EMIT_TILE);
  const int nb = gs.g[ft.pset[f]].nbins, nb_all = nb + PW_NUM_PSEUDO;   // the bins of the frame's parameter set
  const int* bo = bin_off + (size_t) f * (nbp + 1);
  // largest b with bo[b] <= w0: the bin that holds position w0 (empty bins share their offset with the next bin)
  int lo = 0, hi = nb_all;
  while (hi - lo > 1) {
    const int step = (hi - lo + 31) >> 5;
    const int q = lo + lane * step;
    const bool le = q < hi && bo[q] <= w0;
    const unsigned m = __ballot_sync(0xffffffffu, le);   // lane 0 probes lo itself, whose offset is <= w0: m is never empty
    const int k = 31 - __clz(m);
    lo += k * step;
    hi = min(hi, lo + step);
  }
  for (int bb = lo; bb < nb_all; bb += 32) {
    const int b = bb + lane;
    const bool valid = b < nb_all;
    const int off = valid ? bo[b] : n, end = valid ? bo[b + 1] : n;
    const bool need = valid && end > off && off < w1 && end > w0;
    int g_dst = -1, ng_dst = -1, ng = -1;
    if (need) {
      const BinSeg sg = segs[(size_t) f * (gs.nbs + PW_NUM_PSEUDO) + b];
      g_dst = sg.g_dst; ng_dst = sg.ng_dst;
      if (b < nb) { const BinFit& r = fits[(size_t) f * gs.nbs + b]; if (r.fitted) ng = r.n_ground; }
    }
    for (unsigned m = __ballot_sync(0xffffffffu, need); m; m &= m - 1) {
      const int l = __ffs(m) - 1;
      const int o = __shfl_sync(0xffffffffu, off, l), e = __shfl_sync(0xffffffffu, end, l);
      const int gd = __shfl_sync(0xffffffffu, g_dst, l), nd = __shfl_sync(0xffffffffu, ng_dst, l), ngr = __shfl_sync(0xffffffffu, ng, l);
      const int j0 = max(o, w0), j1 = min(e, w1);
      if (ngr >= 0) {
        const int* src = part + p0;
        for (int j = j0 + lane; j < j1; j += 128) {   // four independent loads in flight per lane
          int v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) { const int jj = j + 32 * u; v[u] = src[jj < j1 ? jj : j1 - 1]; }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int jj = j + 32 * u, rel = jj - o;
            if (jj < j1) out_idx[p0 + ((rel < ngr) ? (gd + rel) : (nd + (rel - ngr)))] = v[u];
          }
        }
      } else if (nd >= 0) {   // not fitted: everything to the non-ground list (nd < 0: dropped points, S:591)
        const float4* src = sorted + p0;
        for (int j = j0 + lane; j < j1; j += 32) out_idx[p0 + nd + (j - o)] = __float_as_int(src[j].w);
      }
    }
    if (__ballot_sync(0xffffffffu, valid && off >= w1)) break;   // the window reached the end of the tile
  }
}

// k_gather_xyz: toEigenCloud (S:8-16): xyz of the listed points of one frame.
__global__ void k_gather_xyz(const float4* __restrict__ pts, const int* __restrict__ idx, int n, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float4 p = pts[idx[i]];
    dst[3 * i] = p.x; dst[3 * i + 1] = p.y; dst[3 * i + 2] = p.z;
  }
}

}  // namespace pwpp

// pwpp_front.cuh — the front end of the path as ONE kernel: a THREAD-BLOCK CLUSTER per frame.
//
//   RNR + polar binning      reference reflected_noise_removal S:377-400, pc2czm S:578-622, flush_patches S:33-45
//   per-frame scan + queues  the growth of czm[k][i][j] (S:602-614) and the per-bin gate S:191
//   stable scatter           points of a bin contiguous, ascending point index inside a bin (the order pc2czm produces)
// ("S:" = cpp/patchworkpp/src/patchworkpp.cpp). Results are those of the three stand-alone kernels k_bin_hist / k_bin_scan /
// k_scatter (pwpp_kernels.cuh), which remain as the PWPP_FRONT=0 path; this kernel removes what made them expensive:
//   * the three kernels communicated through global memory (per-chunk histograms and scatter bases: chist / cbase) and
//     each streamed the whole batch, so the cloud was read from HBM twice;
//   * here the 8 CTAs (64 warps) of a cluster split one frame into 64 contiguous slices. Pass 1: every warp bins its slice
//     chunk by chunk — chunks arrive through the TMA engine (cp.async.bulk global -> shared, mbarrier completion, two
//     buffers per warp: SASS UBLKCP) — and counts into its own histogram row in shared memory. After a cluster barrier every
//     CTA reads the other CTAs' histograms through DISTRIBUTED SHARED MEMORY (cluster.map_shared_rank), scans the bins and
//     turns every warp's counts into the warp's first free position of every bin; rank 0 also writes the bin offsets and
//     fills the fit work queues. Pass 2: the warp streams its slice again — 2 MB of a frame read a few microseconds earlier
//     by the same cluster: L2 hits — and scatters. No block barrier and no atomic inside either pass. HBM sees the cloud
//     once (16 B/pt in, 16 B/pt out for the re-laid-out copy, 2 + 2 B/pt of bin ids that mostly stay in L2).
// The bin ids still go to global memory (pwpp_copy_bin_ids, and frames of any size: a dense frame's slice does not fit on chip).
#pragma once
#include "pwpp_common.cuh"
#include "pwpp_fit.cuh"

namespace pwpp {

constexpr int FC_CS = 8;                 // CTAs per cluster (portable maximum)
// Threads per CTA are a template parameter: 256 (64 warps per frame, 4 CTAs per SM) for KITTI-sized frames, 512 (128 warps per frame,
// 2 CTAs per SM) for dense frames whose slices are ten times longer. Of the shapes 8 x 256, 8 x 512 and 4 x 512 CTAs x threads,
// 8 x 512 is the slowest on KITTI-sized frames and the fastest on dense ones.
constexpr int FC_THREADS = 256, FC_THREADS_DENSE = 512;
constexpr int FC_ROWS = 4;               // 32-point rows per chunk
constexpr int FC_CHUNK = FC_ROWS * 32;   // points per TMA chunk of one warp: 2 KB, two buffers per warp in flight

__host__ __device__ inline size_t front_cluster_smem_bytes(int nbp, int nthreads) {
  const int FC_WARPS = nthreads / 32;
  // tiles [FC_WARPS][2][FC_CHUNK] float4 | per-warp counts, later bases [FC_WARPS][nbp] u32 | CTA histogram [nbp] u32 | scan [nbp + 1] i32 (padded to
  // 16 B) | mbarriers [FC_WARPS][2] u64 | class counters [3][NUM_CLASSES] i32
  return (size_t) FC_WARPS * 2 * FC_CHUNK * sizeof(float4) + (size_t) (FC_WARPS + 1) * nbp * sizeof(unsigned) + ((((size_t) nbp + 1) * sizeof(int) + 15) & ~(size_t) 15) +
         (size_t) FC_WARPS * 2 * sizeof(unsigned long long) + 3 * NUM_CLASSES * sizeof(int);
}

// The 64 warps of a cluster split the frame's 32-point rows into 64 CONTIGUOUS slices in (CTA rank, warp) order; a warp walks its
// slice twice, chunk by chunk, and never meets a block barrier while it streams: its chunks arrive in its own two TMA buffers
// (its own mbarriers), it counts into its own histogram row (no atomics: one lane per distinct bin of a row adds), and after the
// scan that row holds the warp's first free position of every bin, which pass 2 advances the same way. A point's position is
// (points of the bin in lower slices) + (points of the bin earlier in this slice) + (lower lanes of the row with the same bin):
// ascending point index inside a bin, as k_scatter produces.
template <bool FAST, int L2MAX, int NT>
__global__ void
#if !defined(PWPP_SIMT_EMU)
__cluster_dims__(FC_CS, 1, 1)
#endif
__launch_bounds__(NT, 1024 / NT) k_front_cluster(const float4* __restrict__ pts, FrameTable ft, const StreamState* __restrict__ states,
                                                  const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps,
                                                  int has_intensity, int nbp, int nbs, unsigned short* __restrict__ bin_ids, int* __restrict__ bin_off, WorkQueues wq,
                                                  BinFit* __restrict__ fits, float4* __restrict__ sorted) {
  constexpr int FC_THREADS = NT, FC_WARPS = NT / 32;   // (shadow the namespace-scope defaults)
  PW_DYN_SHARED(unsigned char, s_raw);
  float4* s_tile = reinterpret_cast<float4*>(s_raw);                                              // [FC_WARPS][2][FC_CHUNK]
  unsigned* s_wb = reinterpret_cast<unsigned*>(s_raw + (size_t) FC_WARPS * 2 * FC_CHUNK * 16);    // [FC_WARPS][nbp] counts of a warp's slice, then its bases
  unsigned* s_hist = s_wb + (size_t) FC_WARPS * nbp;                                              // [nbp] this CTA's bin counts (read by the whole cluster)
  int* s_scan = reinterpret_cast<int*>(s_hist + nbp);                                             // [nbp + 1]
  unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(s_scan) + ((((size_t) nbp + 1) * 4 + 15) & ~(size_t) 15));   // [FC_WARPS][2]
  int* s_cls = reinterpret_cast<int*>(s_bar + FC_WARPS * 2);                                      // [3][NUM_CLASSES]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int f = blockIdx.y;
  const int rank = (int) pw_cluster_rank();
  const long long p0 = ft.pt_off[f];
  const int n = (int) (ft.pt_off[f + 1] - p0);
  const int nrows = (n + 31) >> 5;
  const int gw = rank * FC_WARPS + w;                                                             // slice index in the frame
  const int i0 = (int) ((long long) nrows * gw / (FC_CS * FC_WARPS)) << 5;                        // this warp's points [i0, i1)
  const int i1 = min(n, (int) ((long long) nrows * (gw + 1) / (FC_CS * FC_WARPS)) << 5);
  const float4* fp = pts + p0;
  const int set = ft.pset[f];                                                                     // the frame's parameter set
  const Geometry& g = gs.g[set];
  const AlgoParams& ap = aps.a[set];
  const int nbins = g.nbins;
  const double sensor_height = states[ft.stream[f]].sensor_height;
  const bool rnr_on = ap.enable_RNR && has_intensity;  // S:161, S:379-382
  unsigned* my = s_wb + (size_t) w * nbp;
  float4* my_tile = s_tile + (size_t) w * 2 * FC_CHUNK;
  unsigned long long* my_bar = s_bar + w * 2;

  for (int b = tid; b < FC_WARPS * nbp; b += FC_THREADS) s_wb[b] = 0u;
#if !defined(PWPP_SIMT_EMU)
  if (lane == 0) { mbar_init(&my_bar[0], 1); mbar_init(&my_bar[1], 1); }
  if (tid == 0) asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  __syncthreads();
  unsigned ph = 0u;   // bit b: mbarrier phase of buffer b
  (void) ph;
  auto issue = [&](int c0, int buf) {   // lane 0: points [c0, c0 + FC_CHUNK) of the slice -> buffer buf
#if !defined(PWPP_SIMT_EMU)
    const int cnt = min(FC_CHUNK, i1 - c0);
    fence_proxy_async();
    mbar_expect_tx(&my_bar[buf], (unsigned) cnt * 16u);
    bulk_g2s(my_tile + buf * FC_CHUNK, fp + c0, (unsigned) cnt * 16u, &my_bar[buf]);
#else
    (void) c0; (void) buf;
#endif
  };
  auto wait_chunk = [&](int c0, int buf) {
#if !defined(PWPP_SIMT_EMU)
    (void) c0;
    mbar_wait(&my_bar[buf], (ph >> buf) & 1u);
    ph ^= 1u << buf;
#else
    for (int i = c0 + lane; i < min(c0 + FC_CHUNK, i1); i += 32) my_tile[buf * FC_CHUNK + (i - c0)] = fp[i];
    __syncwarp();
#endif
  };

  // ---------------- pass 1: bin ids + this warp's histogram ----------------
  if (lane == 0 && i0 < i1) issue(i0, 0);
  for (int c0 = i0, buf = 0; c0 < i1; c0 += FC_CHUNK, buf ^= 1) {
    if (lane == 0 && c0 + FC_CHUNK < i1) issue(c0 + FC_CHUNK, buf ^ 1);   // (the warp left that buffer at the __syncwarp that ended the previous chunk)
    wait_chunk(c0, buf);
    const float4* tp = my_tile + buf * FC_CHUNK;
#pragma unroll 2
    for (int r = 0; r < FC_ROWS; ++r) {
      const int i = c0 + r * 32 + lane;
      int bin = -1;
      if (i < i1) {
        const float4 p = tp[r * 32 + lane];
        if (rnr_on && rnr_hit(p.x, p.y, p.z, p.w, sensor_height, ap)) bin = PW_BIN_RNR(g.nbins);
        else if (p.z == FLT_MIN) bin = PW_BIN_DROP(g.nbins);  // S:591
        else bin = FAST ? bin_of_point(p.x, p.y, p.z, g) : bin_of_point_exact(p.x, p.y, p.z, g);
        bin_ids[p0 + i] = (unsigned short) bin;
      }
      const unsigned act = __ballot_sync(0xffffffffu, bin >= 0);
      if (bin >= 0) {   // one lane per distinct bin of the row adds the row's count
        const unsigned peers = __match_any_sync(act, bin);
        if ((peers & lanemask_lt()) == 0) my[bin] += (unsigned) __popc(peers);
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int b = tid; b < nbp; b += FC_THREADS) {
    unsigned t = 0;
#pragma unroll
    for (int ww = 0; ww < FC_WARPS; ++ww) t += s_wb[ww * nbp + b];
    s_hist[b] = t;
  }
  pw_cluster_sync();   // every histogram of the frame is complete and visible cluster-wide

  // ---------------- scan: totals over the cluster, bin offsets, every warp's bases ----------------
  for (int b = tid; b < nbp; b += FC_THREADS) {
    unsigned tot = 0, before = 0;
#pragma unroll
    for (int c = 0; c < FC_CS; ++c) {
      const unsigned h = *pw_cluster_map(&s_hist[b], c);   // distributed shared memory
      if (c < rank) before += h;
      tot += h;
    }
    s_scan[b] = (int) tot;
    reinterpret_cast<unsigned*>(s_tile)[b] = before;   // the tile buffers are idle between the passes: [nbp] "points of the bin in lower CTAs"
  }
  __syncthreads();
  if (tid < 32) {   // exclusive scan over nbp (<= 4096) bins by warp 0
    int carry = 0;
    for (int b0 = 0; b0 < nbp; b0 += 32) {
      const int b = b0 + tid;
      const int v = b < nbp ? s_scan[b] : 0;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (tid >= o) incl += u; }
      if (b < nbp) s_scan[b] = carry + incl - v;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (tid == 0) s_scan[nbp] = carry;
  }
  __syncthreads();
  for (int b = tid; b < nbp; b += FC_THREADS) {   // counts -> first free position of every warp
    unsigned run = (unsigned) s_scan[b] + reinterpret_cast<unsigned*>(s_tile)[b];
#pragma unroll
    for (int ww = 0; ww < FC_WARPS; ++ww) { const unsigned v = s_wb[ww * nbp + b]; s_wb[ww * nbp + b] = run; run += v; }
  }
  pw_cluster_sync();   // nobody reads a remote histogram after this point (a CTA may exit before its neighbours); also orders the reuse of the tile buffers
  if (rank == 0) {
    // what k_bin_scan leaves for the later stages: bin offsets, the fit work queues (S:191: patches below num_min_pts are
    // not fitted), the records of the patches that will not be fitted
    int* bo = bin_off + (size_t) f * (nbp + 1);
    for (int b = tid; b <= nbp; b += FC_THREADS) bo[b] = s_scan[b];
    int* s_cnt = s_cls, *s_cbase = s_cls + NUM_CLASSES, *s_pos = s_cls + 2 * NUM_CLASSES;
    if (tid < NUM_CLASSES) { s_cnt[tid] = 0; s_pos[tid] = 0; }
    __syncthreads();
    auto cls_of = [](int m) { return m <= CLS_S_MAX ? 0 : m <= CLS_M_MAX ? 1 : m <= CLS_L1_MAX ? 2 : m <= L2MAX ? 3 : m <= CLS_L3_MAX ? 4 : 5; };
    for (int b = tid; b < nbins; b += FC_THREADS) {
      const int m = s_scan[b + 1] - s_scan[b];
      if (m >= ap.num_min_pts && m > 0) atomicAdd(&s_cnt[cls_of(m)], 1);
      else {
        BinFit& r = fits[(size_t) f * nbs + b];
        r.n = m; r.n_ground = 0; r.d = 0.0;
        for (int k = 0; k < 3; ++k) { r.mean[k] = 0.0; r.normal[k] = 0.0; r.sv[k] = 0.0; }
        r.fitted = (m >= ap.num_min_pts) ? 1 : 0;   // an EMPTY patch with num_min_pts <= 0 is "fitted" with the previous patch's plane (S:49)
        r.verdict = r.fitted ? PW_FIT_NO_PLANE : 0;
      }
    }
    __syncthreads();
    if (tid < NUM_CLASSES) s_cbase[tid] = s_cnt[tid] ? atomicAdd(&wq.count[tid], s_cnt[tid]) : 0;
    __syncthreads();
    for (int b = tid; b < nbins; b += FC_THREADS) {
      const int m = s_scan[b + 1] - s_scan[b];
      if (m >= ap.num_min_pts && m > 0) {
        const int c = cls_of(m);
        wq.items[c][s_cbase[c] + atomicAdd(&s_pos[c], 1)] = make_work_item(f, b, m, p0 + (long long) s_scan[b]);
      }
    }
  }

  // ---------------- pass 2: stable scatter of this warp's slice ----------------
  float4* out = sorted + p0;
  if (lane == 0 && i0 < i1) issue(i0, 0);
  for (int c0 = i0, buf = 0; c0 < i1; c0 += FC_CHUNK, buf ^= 1) {
    if (lane == 0 && c0 + FC_CHUNK < i1) issue(c0 + FC_CHUNK, buf ^ 1);
    int bins[FC_ROWS];
#pragma unroll
    for (int r = 0; r < FC_ROWS; ++r) { const int i = c0 + r * 32 + lane; bins[r] = (i < i1) ? (int) bin_ids[p0 + i] : -1; }   // written by this very thread in pass 1
    wait_chunk(c0, buf);
    const float4* tp = my_tile + buf * FC_CHUNK;
#pragma unroll
    for (int r = 0; r < FC_ROWS; ++r) {
      const int bin = bins[r];
      const unsigned act = __ballot_sync(0xffffffffu, bin >= 0);
      unsigned peers = 0u, first = 0u;
      if (bin >= 0) { peers = __match_any_sync(act, bin); first = my[bin]; }
      __syncwarp();
      if (bin >= 0) {
        float4 p = tp[r * 32 + lane];
        p.w = __int_as_float(c0 + r * 32 + lane);
        out[first + __popc(peers & lanemask_lt())] = p;
        if ((peers & lanemask_lt()) == 0) my[bin] = first + (unsigned) __popc(peers);
      }
      __syncwarp();
    }
  }
}

}  // namespace pwpp

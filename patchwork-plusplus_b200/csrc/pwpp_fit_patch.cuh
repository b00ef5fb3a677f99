// pwpp_fit_patch.cuh — plane fitting (R-VPF + R-GPF) of ONE LARGE PATCH PER CTA with the patch held in REGISTERS.
//
// Reference: cpp/patchworkpp/src/patchworkpp.cpp ("S:") extract_piecewiseground 467-549, extract_initial_seeds 77-149,
// estimate_plane 47-75, calc_point_to_plane_d 551-554. State machine, arithmetic contract and selection logic are those of
// pwpp_fit.cuh / pwpp_fit_group.cuh; this kernel serves the patches that hold most of the POINTS of a scan (zone 0: 1k..8k
// points each) and is built around what per-warp event traces of the earlier kernels showed: every phase of the
// earlier kernels was bound by the latency of short dependent chains (a shared-memory load, a double conversion, a
// warp-synchronous operation per 32-point row) and by serial sections, not by issue
// slots or bandwidth. Here
//   * a thread loads its SL points ONCE (coalesced 128-bit global loads, all in flight together) and keeps x, y, z in
//     registers; every pass is a fully unrolled, branch-light loop over compile-time slots: no shared-memory traffic, no
//     warp-synchronous operation per row, independent slots overlap in the pipeline;
//   * the threshold tests that the reference does in double ((double) z < t, S:90 / S:108 / S:145) use the float that is
//     exactly equivalent (z < t  <=>  z < round_up_to_float(t) for a float z), so the passes issue FP64 only to accumulate;
//   * the LPR selection needs two barriers: warp-local ranking of the lane minima (32 independent shuffles), the NW x m
//     smallest of them bound the K-th smallest point tightly, the ~K..2K candidates below the bound are ranked exactly;
//   * the 9 moment sums are reduced by an interleaved butterfly (all 9 chains in flight), partials are combined by 9 lanes
//     of warp 0 in warp order (bit-reproducible), the 3x3 problem is solved once (two planes side by side in fused rounds).
#pragma once
#include "pwpp_fit.cuh"
#include "pwpp_trace.cuh"

namespace pwpp {

constexpr int FP_CAND = 128;   // candidates the exact LPR selection handles (4 keys per lane)

// exact selection among cc (<= FP_CAND) candidate keys in cbuf: mean of the `target` smallest (S:99-103) by RANKING: a
// candidate's rank = number of candidates before it in (key, position) order; all compares are independent (no serial
// bisection). The sum of <= 32 floats in double is exact, so the result does not depend on the candidates' order. Uniform.
__device__ __forceinline__ double rank_mean(const unsigned* cbuf, int cc, int target) {
  const int lane = lane_id();
  unsigned ck[FP_CAND / 32];
  int rank[FP_CAND / 32];
  const int nq = (cc + 31) >> 5;
#pragma unroll
  for (int q = 0; q < FP_CAND / 32; ++q) { const int i = lane + 32 * q; ck[q] = i < cc ? cbuf[i] : 0xffffffffu; rank[q] = 0; }
  // candidates are broadcast 8 at a time (independent shared-memory reads in flight); entries past cc hold 0xffffffff (or
  // stale keys) and are masked by the position test
  for (int j0 = 0; j0 < cc; j0 += 8) {
    unsigned v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = cbuf[(j0 + u) < FP_CAND ? (j0 + u) : (FP_CAND - 1)];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int j = j0 + u;
      if (j < cc) {   // uniform
#pragma unroll
        for (int q = 0; q < FP_CAND / 32; ++q) { if (q >= nq) break; rank[q] += (v[u] < ck[q] || (v[u] == ck[q] && j < lane + 32 * q)) ? 1 : 0; }
      }
    }
  }
  double ps = 0.0;
#pragma unroll
  for (int q = 0; q < FP_CAND / 32; ++q) if (lane + 32 * q < cc && rank[q] < target) ps += (double) key_to_float(ck[q]);
  ps = warp_sum(ps);
  return ps / (double) target;
}


constexpr int FP_SL = 16;    // points per thread (register slots)
constexpr int FP_STG = 256;  // staging entries per warp: the participating points of 8 slots

// 9 sums + 2 counts reduced over the warp with all chains in flight (xor butterfly: every lane ends with the totals)
__device__ __forceinline__ void warp_sum9(double (&a)[9], int& c0, int& c1) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double t[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) t[q] = __shfl_xor_sync(0xffffffffu, a[q], o);
    const int u0 = __shfl_xor_sync(0xffffffffu, c0, o), u1 = __shfl_xor_sync(0xffffffffu, c1, o);
#pragma unroll
    for (int q = 0; q < 9; ++q) a[q] += t[q];
    c0 += u0; c1 += u1;
  }
}

// K-th smallest (1-based) of the 32 values held one per lane, by ranking; 0xffffffff entries sort last. Uniform result.
__device__ __forceinline__ unsigned warp_kth_of_32(unsigned v, int K, int& rank_out) {
  const int lane = lane_id();
  int rank = 0;
#pragma unroll
  for (int i = 0; i < 32; ++i) { const unsigned o = __shfl_sync(0xffffffffu, v, i); rank += (o < v || (o == v && i < lane)) ? 1 : 0; }
  rank_out = rank;
  const unsigned holder = __ballot_sync(0xffffffffu, rank == K - 1);
  return __shfl_sync(0xffffffffu, v, __ffs(holder) - 1);
}

// S:525 / S:529 in double for the (rare) points whose fp32 distance lies inside the error bound of th_dist; out of line so that
// the unrolled filter loop stays small
__device__ __noinline__ bool exact_below(float x, float y, float z, const double* plane10, double th) {
  const double dd = dadd(dadd(dadd(dmul(plane10[3], (double) x), dmul(plane10[4], (double) y)), dmul(plane10[5], (double) z)), plane10[9]);
  return dd < th;
}

template <int NW, int MINB, int CLS>
__global__ void __launch_bounds__(NW * 32, MINB) k_fit_patch(const float4* __restrict__ sorted, FrameTable ft, const StreamState* __restrict__ states, const __grid_constant__ GeometrySets gs,
                                                              const __grid_constant__ AlgoParamSets aps, int nbp, const int* __restrict__ bin_off, WorkQueues wq, int* __restrict__ part,
                                                              BinFit* __restrict__ fits) {
  constexpr int NT = NW * 32;
  constexpr int M_TOP = 32 / NW;   // smallest lane minima each warp contributes to the bound
  static_assert(NW == 8 || NW == 16 || NW == 4, "M_TOP * NW == 32");
  __shared__ double s_part[NW][20];      // per-warp partial moments: [0..9) the set, [9] unused, [10..19) inner set of a fused round
  __shared__ int s_pcnt[NW][4];          // per warp: count, inner count / changes, ground, valid
  __shared__ unsigned s_min[NT];            // per-thread minimum key of the LPR candidates
  __shared__ int s_tile[2][FP_SL * NW + 1];   // partition: ground / non-ground count of every (slot, warp) tile, then their exclusive prefix
  __shared__ int s_nv[NW];
  __shared__ unsigned s_cand[FP_CAND];
  __shared__ int s_cc;
  __shared__ double s_plane[10];         // mean[3] normal[3] sv[3] d
  __shared__ double s_tot[10];           // running sums of the R-GPF phase + count
  __shared__ int s_ctl[8];               // 0: solved, 1: taken (fused), 2: changes, 3: n of the fitted set
  __shared__ int4 s_item;
  __shared__ float s_first[2];
  PW_DYN_SHARED(float4, s_stage);   // [NW][FP_STG] compaction buffers of the accumulation
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const unsigned lt = lanemask_lt();
  const int count = wq.count[CLS];
  PW_EV_DECL;

  // queue protocol: the first item is claimed synchronously; afterwards the last warp claims one patch AHEAD (atomic +
  // descriptor load + L2 prefetch of its points while the current patch is processed) and publishes it at the end
  if (tid == 0) {
    const int t = atomicAdd(&wq.head[CLS], 1);
    s_item = t < count ? wq.items[CLS][t] : make_int4(-1, 0, 0, 0);
  }
  for (;;) {
    if (tid == 0) s_cc = 0;
    if (tid < 10) { s_plane[tid] = 0.0; s_tot[tid] = 0.0; }
    __syncthreads();
    PW_EV(1);
    const int4 cur = s_item;
    if (cur.x < 0) return;
    int4 nxt = make_int4(-1, 0, 0, 0);
    if (tid == NT - 32) {   // lane 0 of the last warp
      const int t = atomicAdd(&wq.head[CLS], 1);
      if (t < count) nxt = wq.items[CLS][t];
    }
    const int f = cur.x >> 12, bin = cur.x & 0xfff, n = cur.y;
    const int set = ft.pset[f];                  // the frame's parameter set
    const Geometry& g = gs.g[set];
    const AlgoParams& ap = aps.a[set];
    const float thf = (float) ap.th_dist;
    const bool fuse_ok = ap.th_seeds <= ap.th_seeds_v;
    const int K = ap.num_lpr;
    const long long start = work_item_start(cur);
    const float4* P = sorted + start;
    int* out = part + start;
    const int rpw = (n + NT - 1) / NT;           // slots in use (<= FP_SL): slot k of thread tid is point k * NT + tid, so that
    const int jbase = tid;                         // neighbouring points (similar z within a scan line) land in different threads

    // ---- the patch: SL points per thread, loaded once ----
    float px[FP_SL], py[FP_SL], pz[FP_SL];
    unsigned vmask = 0u;
#pragma unroll
    for (int k = 0; k < FP_SL; ++k) {
      const int j = jbase + k * NT;
      px[k] = 0.f; py[k] = 0.f; pz[k] = 0.f;
      if (k < rpw && j < n) { const float4 q4 = ld_stream_f4(P + j); px[k] = q4.x; py[k] = q4.y; pz[k] = q4.z; vmask |= 1u << k; }
    }
    if (w == NW - 1) {   // the look-ahead warp pulls the next patch towards L2 while this one is processed
      nxt.x = __shfl_sync(0xffffffffu, nxt.x, 0); nxt.y = __shfl_sync(0xffffffffu, nxt.y, 0);
      nxt.z = __shfl_sync(0xffffffffu, nxt.z, 0); nxt.w = __shfl_sync(0xffffffffu, nxt.w, 0);
      if (nxt.x >= 0) prefetch_patch_l2(sorted + work_item_start(nxt), nxt.y, lane, 32);
    }
    PW_EV(2);
    const bool zone0 = bin < g.bin_base[1];
    const double margin_z = ap.adaptive_seed_selection_margin * states[ft.stream[f]].sensor_height;   // S:90
    const float margin_f = zone0 ? float_ru(margin_z) : -INFINITY;                          // (double) z < margin  <=>  z < margin_f
    if (tid == 0) { s_first[0] = px[0]; s_first[1] = py[0]; }   // point 0: reference point of the moment sums (with the LPR height); read after the first barrier of the seed round
    double c0 = 0.0, c1 = 0.0;

    unsigned amask = vmask, member = 0u;
    int state = (ap.enable_RVPF && zone0) ? ST_RVPF : ST_SEED;
    int rvpf_it = 0, gpf_it = 0, n_ground = 0;
    bool have_plane = false;
    double c2 = 0.0;
    float pf0 = 0.f, pf1 = 0.f, pf2 = 0.f, pfd = 0.f;   // float copy of the current plane for the distance filter

    // Moment sums of the slots in `plus` (added) and `minus` (subtracted), relative to (c0, c1, c2). A slot usually holds a
    // point of the set in only some of the 32 lanes, and a double-precision instruction costs the warp several issue cycles
    // whether 1 or 32 lanes take part (event traces: the accumulation was bound by exactly that). So the warp first COMPACTS the
    // participating points of 8 slots into its staging buffer (ballot prefix: slot-major, lane-minor order) and then
    // accumulates full rows of 32: ~3x fewer FP64 instructions in seed rounds, ~10x in late R-GPF rounds.
    float4* stg = s_stage + w * FP_STG;
    auto accumulate = [&](unsigned plus, unsigned minus, double (&acc)[9]) {
      const unsigned any = plus | minus;
#pragma unroll
      for (int k0 = 0; k0 < FP_SL; k0 += 8) {
        if (k0 >= rpw) break;   // uniform
        int cnt = 0;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int k = k0 + u;
          const bool on = (any >> k) & 1u;
          const unsigned bal = __ballot_sync(0xffffffffu, on);
          if (on) stg[cnt + __popc(bal & lt)] = make_float4(px[k], py[k], pz[k], ((minus >> k) & 1u) ? -1.f : 1.f);
          cnt += __popc(bal);
        }
        __syncwarp();
        for (int i0 = 0; i0 < cnt; i0 += 32) {
          const int i = i0 + lane;
          if (i < cnt) {
            const float4 q4 = stg[i];
            const double wgt = (double) q4.w;
            const double dx = (double) q4.x - c0, dy = (double) q4.y - c1, dz = (double) q4.z - c2;
            const double wx = dx * wgt, wy = dy * wgt, wz = dz * wgt;
            acc[0] += wx; acc[1] += wy; acc[2] += wz;
            acc[3] += wx * dx; acc[4] += wx * dy; acc[5] += wx * dz; acc[6] += wy * dy; acc[7] += wy * dz; acc[8] += wz * dz;
          }
        }
        __syncwarp();
      }
    };
    auto accumulate_plus = [&](unsigned plus, double (&acc)[9]) {
#pragma unroll
      for (int k0 = 0; k0 < FP_SL; k0 += 8) {
        if (k0 >= rpw) break;   // uniform
        int cnt = 0;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int k = k0 + u;
          const bool on = (plus >> k) & 1u;
          const unsigned bal = __ballot_sync(0xffffffffu, on);
          if (on) stg[cnt + __popc(bal & lt)] = make_float4(px[k], py[k], pz[k], 1.f);
          cnt += __popc(bal);
        }
        __syncwarp();
        for (int i0 = 0; i0 < cnt; i0 += 32) {
          const int i = i0 + lane;
          if (i < cnt) {
            const float4 q4 = stg[i];
            const double dx = (double) q4.x - c0, dy = (double) q4.y - c1, dz = (double) q4.z - c2;
            acc[0] += dx; acc[1] += dy; acc[2] += dz;
            acc[3] += dx * dx; acc[4] += dx * dy; acc[5] += dx * dz; acc[6] += dy * dy; acc[7] += dy * dz; acc[8] += dz * dz;
          }
        }
        __syncwarp();
      }
    };

    while (state != ST_DONE) {   // uniform across the CTA
      const bool seed_round = state == ST_RVPF || state == ST_SEED;
      const bool fused = fuse_ok && state == ST_RVPF;
      double a[9];
#pragma unroll
      for (int q = 0; q < 9; ++q) a[q] = 0.0;
      PW_EV(10);
      int mn = 0, mx = 0;   // mx: inner count (fused round) or number of membership changes (R-GPF round)
      if (seed_round) {
        // ---- LPR: mean of the K lowest z among the alive points not below the zone-0 margin (S:88-103) ----
        unsigned smask = 0u, kmin = 0xffffffffu;
#pragma unroll
        for (int k = 0; k < FP_SL; ++k) {
          const bool ok = ((amask >> k) & 1u) && !(pz[k] < margin_f);
          if (ok) { smask |= 1u << k; kmin = min(kmin, order_key(pz[k])); }
        }
        int nv = __reduce_add_sync(0xffffffffu, __popc(smask));
        s_min[tid] = kmin;
        if (lane == 0) s_nv[w] = nv;
        PW_EV(11);
        __syncthreads();
        PW_EV(12);
        c0 = (double) s_first[0]; c1 = (double) s_first[1];
        int nvalid = 0;
#pragma unroll
        for (int q = 0; q < NW; ++q) nvalid += s_nv[q];
        const int target = nvalid < K ? nvalid : K;
        // Bound: lane l's minimum over the NW threads (l, l + 32, ...) covers the points == l (mod 32); the K-th smallest of
        // these 32 values (ranked with 32 independent shuffles, no bisection) is >= the K-th smallest point, and because the
        // slot mapping spreads neighbouring points over all lanes only ~1.5 K points lie below it. num_lpr > 32: the
        // K-th smallest of all NT thread minima by bisection.
        unsigned T = 0xffffffffu;
        {
          unsigned mk[NW];
          unsigned lm = 0xffffffffu;
#pragma unroll
          for (int q = 0; q < NW; ++q) { mk[q] = s_min[q * 32 + lane]; lm = min(lm, mk[q]); }
          if (target > 0) {
            if (K <= 32) { int dummy; T = warp_kth_of_32(lm, target, dummy); }
            else {
              int have = 0;
              unsigned kmn = 0xffffffffu, kmx = 0u;
#pragma unroll
              for (int q = 0; q < NW; ++q) if (mk[q] != 0xffffffffu) { ++have; kmn = min(kmn, mk[q]); kmx = max(kmx, mk[q]); }
              have = __reduce_add_sync(0xffffffffu, have);
              if (have >= target) {
                kmn = __reduce_min_sync(0xffffffffu, kmn);
                kmx = __reduce_max_sync(0xffffffffu, kmx);
                T = kth_key(kmn, kmx, target, [&](unsigned cand) {
                  int cnt = 0;
#pragma unroll
                  for (int q = 0; q < NW; ++q) cnt += mk[q] < cand;
                  return __reduce_add_sync(0xffffffffu, cnt);
                });
              }
            }
          }
        }
#pragma unroll
        for (int k = 0; k < FP_SL; ++k) {
          if ((smask >> k) & 1u) {
            const unsigned key = order_key(pz[k]);
            if (key <= T) { const int pos = atomicAdd(&s_cc, 1); if (pos < FP_CAND) s_cand[pos] = key; }
          }
        }
        PW_EV(13);
        __syncthreads();
        PW_EV(14);
        const int cc = s_cc;
#if defined(PWPP_SIMT_EMU) && defined(PWPP_DEBUG_FALLBACK)
        if (tid == 0) std::fprintf(stderr, "sel: n=%d cc=%d target=%d\n", n, cc, target);
#endif
        double lpr = 0.0;   // S:99-103 with no candidate: lpr_height stays 0
        if (target > 0) {
          if (cc <= FP_CAND) lpr = rank_mean(s_cand, cc, target);   // every warp, redundantly: no third barrier
          else {
            // rare: num_lpr > 32 or more than FP_CAND points tie below the bound: CTA-wide bisection on the order keys
#if defined(PWPP_SIMT_EMU) && defined(PWPP_DEBUG_FALLBACK)
            if (tid == 0) std::fprintf(stderr, "fallback: n=%d cc=%d target=%d T=%08x nvalid=%d\n", n, cc, target, T, nvalid);
#endif
            unsigned ans = 0u;
            for (int bit = 31; bit >= 0; --bit) {
              const unsigned cand = ans | (1u << bit);
              int cnt = 0;
#pragma unroll
              for (int k = 0; k < FP_SL; ++k) cnt += (((smask >> k) & 1u) && order_key(pz[k]) < cand) ? 1 : 0;
              cnt = __reduce_add_sync(0xffffffffu, cnt);
              __syncthreads();
              if (lane == 0) s_nv[w] = cnt;
              __syncthreads();
              int tot = 0;
#pragma unroll
              for (int q = 0; q < NW; ++q) tot += s_nv[q];
              if (tot < target) ans = cand;
            }
            double ps = 0.0;
            int c_lt = 0;
#pragma unroll
            for (int k = 0; k < FP_SL; ++k) if (((smask >> k) & 1u) && order_key(pz[k]) < ans) { ps += (double) pz[k]; ++c_lt; }
            ps = warp_sum(ps);
            c_lt = __reduce_add_sync(0xffffffffu, c_lt);
            __syncthreads();
            if (lane == 0) { s_part[w][0] = ps; s_nv[w] = c_lt; }
            __syncthreads();
            double tps = 0.0;
            int tlt = 0;
#pragma unroll
            for (int q = 0; q < NW; ++q) { tps += s_part[q][0]; tlt += s_nv[q]; }
            lpr = (tps + (double) (target - tlt) * (double) key_to_float(ans)) / (double) target;
          }
        }
        c2 = lpr;
        PW_EV(15);
        // ---- seeds {alive, z < lpr + th} (S:107-111 / S:144-148); a fused R-VPF round also the inner set of the R-GPF seed fit ----
        const float zthr_f = float_ru(lpr + (state == ST_RVPF ? ap.th_seeds_v : ap.th_seeds)), zin_f = float_ru(lpr + ap.th_seeds);
        unsigned sel = 0u, seli = 0u;
#pragma unroll
        for (int k = 0; k < FP_SL; ++k) {
          const bool in = ((amask >> k) & 1u) && pz[k] < zthr_f;
          sel |= (in ? 1u : 0u) << k;
          seli |= ((in && pz[k] < zin_f) ? 1u : 0u) << k;
        }
        member = fused ? seli : sel;
        accumulate_plus(fused ? (sel & ~seli) : sel, a);   // fused: the seeds outside the inner set; the solver adds the inner sums
        mn = __popc(fused ? (sel & ~seli) : sel);
        if (fused) {   // the inner set in a second sweep over the registers
          warp_sum9(a, mn, mx);
          if (lane == 0) {
#pragma unroll
            for (int q = 0; q < 9; ++q) s_part[w][q] = a[q];
            s_pcnt[w][0] = mn;
          }
#pragma unroll
          for (int q = 0; q < 9; ++q) a[q] = 0.0;
          accumulate_plus(seli, a);
          mn = __popc(seli);
          mx = 0;
        }
      } else {
        // ---- R-GPF round (S:516-543), incremental: only points whose membership changed touch the sums ----
        unsigned inm = 0u;
        if (have_plane) {
#pragma unroll
          for (int k = 0; k < FP_SL; ++k) {
            if (k >= rpw) break;   // uniform
            const float sf = fmaf(pf0, px[k], fmaf(pf1, py[k], fmaf(pf2, pz[k], pfd)));
            const float bound = 1e-6f * (fabsf(px[k]) + fabsf(py[k]) + fabsf(pz[k]) + fabsf(pfd) + 1.0f);   // rigorous fp32 error bound, see dist_filter
            const float diff = sf - thf;
            bool in = diff < 0.f;
            if (!(fabsf(diff) > bound)) in = exact_below(px[k], py[k], pz[k], s_plane, ap.th_dist);
            inm |= (in ? 1u : 0u) << k;
          }
        }
        inm &= amask;
        const unsigned chg = inm ^ member;
        member = inm;
        accumulate(chg & inm, chg & ~inm, a);
        mn = __popc(chg & inm) - __popc(chg & ~inm);
        mx = __popc(chg);
      }
      PW_EV(20);
      // ---- combine: warp butterfly, then 9 (18) lanes of warp 0 add the NW partials in warp order ----
      warp_sum9(a, mn, mx);
      if (lane == 0) {
        if (fused) {   // (the outer set's partial was stored above)
#pragma unroll
          for (int q = 0; q < 9; ++q) s_part[w][10 + q] = a[q];
          s_pcnt[w][1] = mn;
        } else {
#pragma unroll
          for (int q = 0; q < 9; ++q) s_part[w][q] = a[q];
          s_pcnt[w][0] = mn; s_pcnt[w][1] = mx;
        }
      }
      PW_EV(21);
      __syncthreads();
      PW_EV(22);
      if (w == 0) {
        const int ql = lane & 15;
        const bool hi = lane >= 16;
        double v = 0.0;
        int cn = 0;
        if (ql < 9) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) v += s_part[ww][(hi ? 10 : 0) + ql];
          if (fused && !hi) {   // all seeds = the seeds outside the inner set + the inner set
#pragma unroll
            for (int ww = 0; ww < NW; ++ww) v += s_part[ww][10 + ql];
          }
        } else if (ql == 9) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) cn += s_pcnt[ww][hi ? 1 : 0];
          if (fused && !hi) {
#pragma unroll
            for (int ww = 0; ww < NW; ++ww) cn += s_pcnt[ww][1];
          }
        }
        // lanes 0..15: the set of this round; lanes 16..31: the inner set (fused) / the change count
        Moments m;
        const int basel = hi ? 16 : 0;
#pragma unroll
        for (int q = 0; q < 3; ++q) m.s1[q] = __shfl_sync(0xffffffffu, v, basel + q);
#pragma unroll
        for (int q = 0; q < 6; ++q) m.s2[q] = __shfl_sync(0xffffffffu, v, basel + 3 + q);
        m.n = __shfl_sync(0xffffffffu, cn, basel + 9);
        const int other_n = __shfl_sync(0xffffffffu, cn, (hi ? 0 : 16) + 9);   // lanes < 16: inner count / changes
        bool refit = true;
        if (!seed_round) {
          const int changed = other_n;   // (lanes >= 16 do not matter in R-GPF rounds)
          if (changed == 0) refit = false;   // fixpoint
          else {
#pragma unroll
            for (int q = 0; q < 3; ++q) m.s1[q] += s_tot[q];
#pragma unroll
            for (int q = 0; q < 6; ++q) m.s2[q] += s_tot[3 + q];
            m.n += (int) s_tot[9];
          }
          if (lane == 0) s_ctl[2] = changed;
        }
        PW_EV(23);
        const int totn = refit ? m.n : (int) s_tot[9];
        if (tid == 0) s_cc = 0;   // (every warp has read the candidate count of this round's selection)
        Plane mine;
        bool solved = false;
        if (refit && m.n > 0 && (!hi || fused)) {
          const double cc3[3] = {c0, c1, c2};
          plane_from_moments(m, cc3, mine);
          solved = true;
        }
        PW_EV(24);
        __syncwarp();   // every lane has read s_tot / s_plane before lanes 0 / 16 rewrite them
        if (fused) {
          // lane 0 holds the R-VPF plane (all seeds), lane 16 the R-GPF seed plane (inner seeds)
          const double vz_new = __shfl_sync(0xffffffffu, mine.normal[2], 0);
          const bool solved0 = __shfl_sync(0xffffffffu, solved ? 1 : 0, 0) != 0;
          const bool hv = have_plane || solved0;
          const double vz = solved0 ? vz_new : s_plane[5];
          const bool taken = !(hv && vz < ap.uprightness_thr);   // S:489 false -> S:506 break: nothing removed, the seed fit follows
          const int src = (taken && __shfl_sync(0xffffffffu, solved ? 1 : 0, 16) != 0) ? 16 : 0;
          const bool pub = src == 16 ? true : solved0;
          if (lane == src && pub) {
#pragma unroll
            for (int q = 0; q < 3; ++q) { s_plane[q] = mine.mean[q]; s_plane[3 + q] = mine.normal[q]; s_plane[6 + q] = mine.sv[q]; }
            s_plane[9] = mine.d;
          }
          // the R-VPF plane decides about the removal even when the seed plane is published: keep it for the removal pass
          if (lane == (taken ? 16 : 0)) {
#pragma unroll
            for (int q = 0; q < 3; ++q) s_tot[q] = m.s1[q];
#pragma unroll
            for (int q = 0; q < 6; ++q) s_tot[3 + q] = m.s2[q];
            s_tot[9] = (double) m.n;
            s_ctl[3] = m.n;
          }
          if (lane == 0) { s_ctl[0] = (solved0 || (taken && src == 16)) ? 1 : 0; s_ctl[1] = taken ? 1 : 0; }
        } else if (lane == 0) {
          if (refit) {
#pragma unroll
            for (int q = 0; q < 3; ++q) s_tot[q] = m.s1[q];
#pragma unroll
            for (int q = 0; q < 6; ++q) s_tot[3 + q] = m.s2[q];
            s_tot[9] = (double) m.n;
          }
          if (solved) {
#pragma unroll
            for (int q = 0; q < 3; ++q) { s_plane[q] = mine.mean[q]; s_plane[3 + q] = mine.normal[q]; s_plane[6 + q] = mine.sv[q]; }
            s_plane[9] = mine.d;
          }
          s_ctl[0] = solved ? 1 : 0; s_ctl[1] = 0; s_ctl[3] = totn;
        }
      }
      PW_EV(25);
      __syncthreads();
      PW_EV(26);
      // ---- state transition (same machine as k_fit_cta), every thread ----
      if (s_ctl[0]) have_plane = true;   // S:49: an empty set keeps the previous plane
      const int tot_n = s_ctl[3];
      pf0 = (float) s_plane[3]; pf1 = (float) s_plane[4]; pf2 = (float) s_plane[5]; pfd = (float) s_plane[9];
      bool removal = false;
      if (fused) {
        if (s_ctl[1]) { state = (ap.num_iter > 1) ? ST_GPF : ST_FINAL; gpf_it = 0; }
        else { removal = true; ++rvpf_it; if (rvpf_it >= ap.num_iter) state = ST_SEED; }
      } else if (state == ST_RVPF) {
        if (have_plane && s_plane[5] < ap.uprightness_thr) { removal = true; ++rvpf_it; if (rvpf_it >= ap.num_iter) state = ST_SEED; }
        else state = ST_SEED;   // S:506 break
      } else if (state == ST_SEED) {
        state = (ap.num_iter > 1) ? ST_GPF : ST_FINAL;
        gpf_it = 0;
      } else if (state == ST_GPF) {
        ++gpf_it;
        if (gpf_it >= ap.num_iter - 1) state = ST_FINAL;
        if (s_ctl[2] == 0) state = ST_DONE;   // fixpoint: every later iteration reproduces this set and this plane
      } else state = ST_DONE;   // ST_FINAL
      if (removal) {   // S:495-504: points within th_dist_v of the vertical plane leave the patch (exact distance)
        Plane rp;
#pragma unroll
        for (int q = 0; q < 3; ++q) { rp.mean[q] = s_plane[q]; rp.normal[q] = s_plane[3 + q]; rp.sv[q] = s_plane[6 + q]; }
        rp.d = s_plane[9];
#pragma unroll
        for (int k = 0; k < FP_SL; ++k)
          if (((amask >> k) & 1u) && fabs(point_plane_distance(rp, px[k], py[k], pz[k])) < ap.th_dist_v) {   // S:499
            amask &= ~(1u << k);
            if (wq.labels) wq.labels[start + jbase + k * NT] = (unsigned char) rvpf_it;   // (rvpf_it was incremented above: 1-based)
          }
      }
      if (state == ST_DONE) n_ground = have_plane ? tot_n : 0;
    }
    PW_EV(30);
    const unsigned gmask = have_plane ? member : 0u;

    // ---- stable partition: ground indices ascending, then non-ground indices ascending ----
    // point k * NT + tid: tile (k, w) holds 32 consecutive points; the tiles' counts are scanned in (k, w) order
    {
      int idxv[FP_SL];
#pragma unroll
      for (int k = 0; k < FP_SL; ++k) idxv[k] = ((vmask >> k) & 1u) ? reinterpret_cast<const int*>(P)[4 * (jbase + k * NT) + 3] : 0;   // all loads in flight (L2 hits)
      unsigned bgk[FP_SL], bnk[FP_SL];
#pragma unroll
      for (int k = 0; k < FP_SL; ++k) {
        bgk[k] = 0u; bnk[k] = 0u;
        if (k < rpw) {   // uniform
          const bool v = (vmask >> k) & 1u, isg = v && ((gmask >> k) & 1u);
          bgk[k] = __ballot_sync(0xffffffffu, isg);
          bnk[k] = __ballot_sync(0xffffffffu, v && !isg);
          if (lane == 0) { s_tile[0][k * NW + w] = __popc(bgk[k]); s_tile[1][k * NW + w] = __popc(bnk[k]); }
        }
      }
      PW_EV(31);
      __syncthreads();
      PW_EV(32);
      if (w < 2) {   // warp 0: ground counts, warp 1: non-ground counts -> exclusive prefix over the rpw * NW tiles
        const int nt = rpw * NW;
        int carry = 0;
        for (int t0 = 0; t0 < nt; t0 += 32) {
          const int t = t0 + lane;
          const int v = t < nt ? s_tile[w][t] : 0;
          int incl = v;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
          if (t < nt) s_tile[w][t] = carry + incl - v;
          carry += __shfl_sync(0xffffffffu, incl, 31);
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < FP_SL; ++k) {
        if (k < rpw && ((vmask >> k) & 1u)) {
          const bool isg = (gmask >> k) & 1u;
          if (isg) out[s_tile[0][k * NW + w] + __popc(bgk[k] & lt)] = idxv[k];
          else out[n_ground + s_tile[1][k * NW + w] + __popc(bnk[k] & lt)] = idxv[k];
          if (wq.labels && (isg || ((amask >> k) & 1u))) wq.labels[start + jbase + k * NT] = isg ? PW_LABEL_GROUND : PW_LABEL_REJECT;
        }
      }
      if (tid == 0) {
        BinFit& r = fits[(size_t) f * gs.nbs + bin];
        r.n = n; r.n_ground = n_ground; r.fitted = 1;
        r.verdict = have_plane ? 0 : PW_FIT_NO_PLANE;
#pragma unroll
        for (int q = 0; q < 3; ++q) { r.mean[q] = s_plane[q]; r.normal[q] = s_plane[3 + q]; r.sv[q] = s_plane[6 + q]; }
        r.d = s_plane[9];
      }
    }
    __syncthreads();   // every thread is done with s_item / the tables of this patch
    if (tid == NT - 32) s_item = nxt;
  }
}

}  // namespace pwpp

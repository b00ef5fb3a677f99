// pwpp_fit_big.cuh — plane fitting for class X patches (more than 8192 points: dense sensors, BASELINE config 5).
//
// Same per-patch algorithm and citations as pwpp_fit.cuh (reference cpp/patchworkpp/src/patchworkpp.cpp "S:":
// extract_piecewiseground 467-549, extract_initial_seeds 77-149, estimate_plane 47-75). A patch of this size does not
// fit the register / shared-memory resident kernels, and one warp per patch would leave a 1M-point frame's
// thirty-odd 20k..40k-point patches on thirty-odd warps. Here one CTA owns a patch: every pass streams the patch from
// L2 (it was written by k_scatter just before and is re-read 5..7 times; 16 B x 40k points = 640 KB stays L2-resident)
// with NT-strided, fully coalesced float4 loads, four in flight per thread; per-pass state is recomputed instead of
// stored (alive = not removed by a stored R-VPF plane, S:495-504; ground = below the classification plane, S:529),
// so a patch of any size needs no per-point storage.
//   * LPR height: two-level selection like k_fit_cta — the num_lpr-th smallest of the NT per-thread minima bounds the
//     num_lpr-th smallest point; the few points not above it are gathered in shared memory and selected exactly by
//     warp 0. Ties beyond the buffer fall back to a CTA-wide bisection over the patch.
//   * moments: per-thread double sums -> warp butterfly -> warp 0 adds the NW partials in a fixed order
//     (bit-reproducible run to run) and solves the 3x3 problem.
//   * FUSE (see k_fit_warp): an R-VPF round also accumulates the R-GPF seed set and warp 0 solves both planes in its
//     two halves; an upright R-VPF plane (the common case) then skips the separate seed round.
//   * stable partition (ground ascending, then non-ground ascending, like every fit kernel): NT-point tiles, one
//     barrier per tile (double-buffered per-warp counts).
#pragma once
#include "pwpp_fit.cuh"

namespace pwpp {

constexpr int BIG_CCAP = 512;   // candidate buffer of the LPR selection (16 keys per lane of warp 0)
constexpr int BIG_U = 4;        // loads in flight per thread (on dense frames 2 in flight was slower, 8 no faster)

template <int NW, int MINB, bool FUSE>
__global__ void __launch_bounds__(NW * 32, MINB) k_fit_big(const float4* __restrict__ sorted, FrameTable ft, const StreamState* __restrict__ states, const __grid_constant__ GeometrySets gs,
                                                            const __grid_constant__ AlgoParamSets aps, int nbp, const int* __restrict__ bin_off, WorkQueues wq, int* __restrict__ part,
                                                            BinFit* __restrict__ fits) {
  constexpr int NT = NW * 32;
  constexpr int CLS = NUM_CLASSES - 1;
  static_assert(NW == 8 || NW == 16 || NW == 32, "warp 0 keeps NW per-thread minima per lane");
  __shared__ double s_part[NW][18];   // per-warp partial moments: [0..9) all seeds / selected points, [9..18) inner seeds (FUSE)
  __shared__ int s_pcnt[NW][2];
  __shared__ unsigned s_min[NT];
  __shared__ unsigned s_cand[BIG_CCAP];
  __shared__ int s_wcnt[2][NW][2];
  __shared__ unsigned s_u[NW][2];
  __shared__ double s_fb[NW];
  __shared__ double s_lpr;
  __shared__ unsigned s_T;
  __shared__ int s_ccount;
  __shared__ int s_n[2];
  __shared__ Plane s_plane, s_plane2;
  __shared__ int4 s_item;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const unsigned lt = lanemask_lt();

  for (;;) {
    if (tid == 0) {
      const int t = atomicAdd(&wq.head[CLS], 1);
      s_item = t < wq.count[CLS] ? wq.items[CLS][t] : make_int4(-1, 0, 0, 0);
    }
    __syncthreads();
    const int4 cur = s_item;
    if (cur.x < 0) return;
    const int f = cur.x >> 12, bin = cur.x & 0xfff, n = cur.y;
    const int set = ft.pset[f];                  // the frame's parameter set
    const Geometry& g = gs.g[set];
    const AlgoParams& ap = aps.a[set];
    const float thf = (float) ap.th_dist;
    const bool fuse_ok = FUSE && (ap.th_seeds <= ap.th_seeds_v);
    const long long start = work_item_start(cur);
    const float4* P = sorted + start;
    int* out = part + start;
    const int zone = (bin >= g.bin_base[3]) ? 3 : (bin >= g.bin_base[2]) ? 2 : (bin >= g.bin_base[1]) ? 1 : 0;
    const bool zone0 = (zone == 0);
    // S:90; (double) z < margin  <=>  z < margin_f (float_ru), folded with the zone-0 condition
    const float margin_f = zone0 ? float_ru(ap.adaptive_seed_selection_margin * states[ft.stream[f]].sensor_height) : -INFINITY;

    RvpfPlanes rv;
    rv.n = 0;
    Plane pl;
    pl.d = 0.0;
#pragma unroll
    for (int q = 0; q < 3; ++q) { pl.mean[q] = 0.0; pl.normal[q] = 0.0; pl.sv[q] = 0.0; }
    bool have_plane = false;
    const float4 first = P[0];
    double c[3] = {(double) first.x, (double) first.y, 0.0};

    // candidate of the LPR selection: alive and, in zone 0, not below the adaptive margin (S:88-96)
    auto lpr_valid = [&](const float4& p) {
      bool v = (rv.n == 0) || is_alive(rv, ap.th_dist_v, p.x, p.y, p.z);
      if (p.z < margin_f) v = false;
      return v;
    };

    // ---- LPR height: mean of the (<= num_lpr) lowest z among the candidates (S:99-103). Uniform result. ----
    auto select_lpr = [&]() -> double {
      unsigned kmin = 0xffffffffu, kmax = 0u;
      int nv = 0;
      for (int i0 = tid; i0 < n; i0 += BIG_U * NT) {
        float4 q[BIG_U];
#pragma unroll
        for (int u = 0; u < BIG_U; ++u) { const int j = i0 + u * NT; q[u] = P[j < n ? j : n - 1]; }
#pragma unroll
        for (int u = 0; u < BIG_U; ++u) {
          const int j = i0 + u * NT;
          if (j < n && lpr_valid(q[u])) { const unsigned key = order_key(q[u].z); kmin = min(kmin, key); kmax = max(kmax, key); ++nv; }
        }
      }
      s_min[tid] = kmin;
      nv = __reduce_add_sync(0xffffffffu, nv);
      const unsigned wmn = __reduce_min_sync(0xffffffffu, kmin), wmx = __reduce_max_sync(0xffffffffu, kmax);
      if (lane == 0) { s_pcnt[w][0] = nv; s_u[w][0] = wmn; s_u[w][1] = wmx; }
      if (tid == 0) s_ccount = 0;
      __syncthreads();
      int nvalid = 0;
      unsigned amn = 0xffffffffu, amx = 0u;
#pragma unroll
      for (int q = 0; q < NW; ++q) { nvalid += s_pcnt[q][0]; amn = min(amn, s_u[q][0]); amx = max(amx, s_u[q][1]); }
      const int target = nvalid < ap.num_lpr ? nvalid : ap.num_lpr;
      if (target == 0) { __syncthreads(); return 0.0; }   // S:99-103 with no candidate: lpr_height stays 0
      if (w == 0) {
        unsigned mk[NW];
        int have = 0;
#pragma unroll
        for (int q = 0; q < NW; ++q) { mk[q] = s_min[lane * NW + q]; have += mk[q] != 0xffffffffu; }
        have = __reduce_add_sync(0xffffffffu, have);
        unsigned ans = 0xffffffffu;   // fewer candidate-holding threads than target: keep everything
        if (have >= target) {
          unsigned kmn = 0xffffffffu, kmx = 0u;
#pragma unroll
          for (int q = 0; q < NW; ++q) if (mk[q] != 0xffffffffu) { kmn = min(kmn, mk[q]); kmx = max(kmx, mk[q]); }
          kmn = __reduce_min_sync(0xffffffffu, kmn);
          kmx = __reduce_max_sync(0xffffffffu, kmx);
          ans = kth_key(kmn, kmx, target, [&](unsigned cand) {
            int cnt = 0;
#pragma unroll
            for (int q = 0; q < NW; ++q) cnt += mk[q] < cand;
            return __reduce_add_sync(0xffffffffu, cnt);
          });
        }
        if (lane == 0) s_T = ans;
      }
      __syncthreads();
      const unsigned T = s_T;
      for (int i0 = tid; i0 < n; i0 += BIG_U * NT) {
        float4 q[BIG_U];
#pragma unroll
        for (int u = 0; u < BIG_U; ++u) { const int j = i0 + u * NT; q[u] = P[j < n ? j : n - 1]; }
#pragma unroll
        for (int u = 0; u < BIG_U; ++u) {
          const int j = i0 + u * NT;
          if (j < n && lpr_valid(q[u])) {
            const unsigned key = order_key(q[u].z);
            if (key <= T) { const int pos = atomicAdd(&s_ccount, 1); if (pos < BIG_CCAP) s_cand[pos] = key; }
          }
        }
      }
      __syncthreads();
      const int cc = s_ccount;
      if (cc <= BIG_CCAP) {
        if (w == 0) {   // exact selection among the gathered candidates (their order in s_cand does not matter)
          unsigned ck[BIG_CCAP / 32];
          unsigned kmn = 0xffffffffu, kmx = 0u;
          const int nq = (cc + 31) >> 5;
#pragma unroll
          for (int q = 0; q < BIG_CCAP / 32; ++q) {
            const int i = lane + 32 * q;
            ck[q] = i < cc ? s_cand[i] : 0xffffffffu;
            if (i < cc) { kmn = min(kmn, ck[q]); kmx = max(kmx, ck[q]); }
          }
          kmn = __reduce_min_sync(0xffffffffu, kmn);
          kmx = __reduce_max_sync(0xffffffffu, kmx);
          const unsigned ans = kth_key(kmn, kmx, target, [&](unsigned cand) {
            int cnt = 0;
#pragma unroll
            for (int q = 0; q < BIG_CCAP / 32; ++q) { if (q >= nq) break; cnt += ck[q] < cand; }
            return __reduce_add_sync(0xffffffffu, cnt);
          });
          double ps = 0.0;
          int c_lt = 0;
#pragma unroll
          for (int q = 0; q < BIG_CCAP / 32; ++q) if (ck[q] < ans) { ps += (double) key_to_float(ck[q]); ++c_lt; }
          ps = warp_sum(ps);
          c_lt = __reduce_add_sync(0xffffffffu, c_lt);
          if (lane == 0) s_lpr = (ps + (double) (target - c_lt) * (double) key_to_float(ans)) / (double) target;
        }
        __syncthreads();
      } else {
        // many ties at the bound (a perfectly flat synthetic plane): CTA-wide bisection over the whole patch, started
        // below the bits all candidate keys share
        unsigned ans = amn;
        const unsigned diff = amn ^ amx;
        if (diff != 0u) {
          const int top = 31 - __clz(diff);
          ans = (top == 31) ? 0u : (amn & ~((2u << top) - 1u));
          for (int bit = top; bit >= 0; --bit) {
            const unsigned cand = ans | (1u << bit);
            int cnt = 0;
            for (int i = tid; i < n; i += NT) { const float4 p = P[i]; if (lpr_valid(p) && order_key(p.z) < cand) ++cnt; }
            cnt = __reduce_add_sync(0xffffffffu, cnt);
            if (lane == 0) s_pcnt[w][1] = cnt;
            __syncthreads();
            int tot = 0;
#pragma unroll
            for (int q = 0; q < NW; ++q) tot += s_pcnt[q][1];
            __syncthreads();
            if (tot < target) ans = cand;
          }
        }
        double ps = 0.0;
        int c_lt = 0;
        for (int i = tid; i < n; i += NT) { const float4 p = P[i]; if (lpr_valid(p) && order_key(p.z) < ans) { ps += (double) p.z; ++c_lt; } }
        ps = warp_sum(ps);
        c_lt = __reduce_add_sync(0xffffffffu, c_lt);
        if (lane == 0) { s_fb[w] = ps; s_pcnt[w][1] = c_lt; }
        __syncthreads();
        if (tid == 0) {
          double tps = 0.0;
          int tlt = 0;
          for (int q = 0; q < NW; ++q) { tps += s_fb[q]; tlt += s_pcnt[q][1]; }
          s_lpr = (tps + (double) (target - tlt) * (double) key_to_float(ans)) / (double) target;
        }
        __syncthreads();
      }
      return s_lpr;
    };

    // ---- one pass + plane fit. MODE 0: seeds {alive, z < zthr} (FUSED: also the inner set {z < zin}; both float_ru of the
    //      double thresholds);
    //      MODE 1: {alive, signed distance to `cls` < th_dist}. Leaves the counts in nsel[0..1] and, for non-empty
    //      sets, the fitted planes in s_plane / s_plane2 (valid until the next call). ----
    int nsel[2] = {0, 0};
    auto fit_pass = [&](int mode, bool fused, float zthr, float zin, const Plane& cls, const double cc[3]) {
      double a[9], b[FUSE ? 9 : 1];
#pragma unroll
      for (int q = 0; q < 9; ++q) a[q] = 0.0;
#pragma unroll
      for (int q = 0; q < (FUSE ? 9 : 1); ++q) b[q] = 0.0;
      int na = 0, nb = 0;
      PlaneF pf;
      pf.n0 = (float) cls.normal[0]; pf.n1 = (float) cls.normal[1]; pf.n2 = (float) cls.normal[2]; pf.d = (float) cls.d;
      for (int i0 = tid; i0 < n; i0 += BIG_U * NT) {
        float4 q[BIG_U];
#pragma unroll
        for (int u = 0; u < BIG_U; ++u) { const int j = i0 + u * NT; q[u] = P[j < n ? j : n - 1]; }
#pragma unroll
        for (int u = 0; u < BIG_U; ++u) {
          const int j = i0 + u * NT;
          const float4 p = q[u];
          bool in = j < n;
          if (in && rv.n != 0) in = is_alive(rv, ap.th_dist_v, p.x, p.y, p.z);
          if (mode == 0) in = in && (p.z < zthr);                                            // S:108 / S:145
          else if (in) {
            int fl = dist_filter(pf, thf, p.x, p.y, p.z);
            if (fl < 0) fl = (point_plane_distance(cls, p.x, p.y, p.z) < ap.th_dist) ? 1 : 0;   // S:525 / S:529, exact
            in = fl != 0;
          }
          if (in) {
            const double dx = (double) p.x - cc[0], dy = (double) p.y - cc[1], dz = (double) p.z - cc[2];
            a[0] += dx; a[1] += dy; a[2] += dz;
            a[3] += dx * dx; a[4] += dx * dy; a[5] += dx * dz; a[6] += dy * dy; a[7] += dy * dz; a[8] += dz * dz;
            ++na;
            if (FUSE && fused && (p.z < zin)) {
              b[0] += dx; b[1] += dy; b[2] += dz;
              b[3] += dx * dx; b[4] += dx * dy; b[5] += dx * dz; b[6] += dy * dy; b[7] += dy * dz; b[8] += dz * dz;
              ++nb;
            }
          }
        }
      }
      // warp sums by reduce-scatter (pwpp_fit.cuh): the lane that ends up holding quantity q stores it
      na = __reduce_add_sync(0xffffffffu, na);
      if (FUSE && fused) {
        double v[18];
#pragma unroll
        for (int q = 0; q < 9; ++q) { v[q] = a[q]; v[9 + q] = b[FUSE ? q : 0]; }
        reduce_scatter<18, 16>(v, lane);
#pragma unroll
        for (int q = 0; q < 18; ++q)
          if (lane == rs_lane(18, 16, q)) s_part[w][q] = v[rs_slot(18, 16, q)];
        nb = __reduce_add_sync(0xffffffffu, nb);
      } else {
        reduce_scatter<9, 16>(a, lane);
#pragma unroll
        for (int q = 0; q < 9; ++q)
          if (lane == rs_lane(9, 16, q)) s_part[w][q] = a[rs_slot(9, 16, q)];
      }
      if (lane == 0) {
        s_pcnt[w][0] = na;
        if (FUSE && fused) s_pcnt[w][1] = nb;
      }
      __syncthreads();
      if (w == 0) {
        // lanes 0..8 (16..24) add the NW partials of quantity q of the first (inner) set in warp order; lane 9 (25) the counts
        const int ql = lane & 15;
        const bool hi = lane >= 16;
        const bool mine_used = !hi || (FUSE && fused);
        double v = 0.0;
        int cn = 0;
        if (mine_used && ql < 9) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) v += s_part[ww][(hi ? 9 : 0) + ql];
        } else if (mine_used && ql == 9) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) cn += s_pcnt[ww][hi ? 1 : 0];
        }
        const int half = (FUSE && fused && hi) ? 16 : 0;   // without fusion every lane solves the one plane
        Moments ms;
#pragma unroll
        for (int q = 0; q < 3; ++q) ms.s1[q] = __shfl_sync(0xffffffffu, v, half + q);
#pragma unroll
        for (int q = 0; q < 6; ++q) ms.s2[q] = __shfl_sync(0xffffffffu, v, half + 3 + q);
        ms.n = __shfl_sync(0xffffffffu, cn, half + 9);
        Plane mine = pl;
        if (ms.n > 0) plane_from_moments(ms, cc, mine);
        if (lane == 0) { s_plane = mine; s_n[0] = ms.n; }
        if (lane == 16) { s_plane2 = mine; s_n[1] = (FUSE && fused) ? ms.n : 0; }
      }
      __syncthreads();
      nsel[0] = s_n[0];
      nsel[1] = s_n[1];
    };

    // 1. R-VPF (S:482-508). For zone != 0 the fitted plane can never be used (see k_fit_stream).
    bool seed_done = false;
    if (ap.enable_RVPF && zone0) {
      for (int it = 0; it < ap.num_iter; ++it) {
        const double lpr = select_lpr();
        c[2] = lpr;
        fit_pass(0, fuse_ok, float_ru(lpr + ap.th_seeds_v), float_ru(lpr + ap.th_seeds), pl, c);
        if (nsel[0] > 0) { pl = s_plane; have_plane = true; }
        if (have_plane && pl.normal[2] < ap.uprightness_thr) {  // S:489
          if (rv.n < MAX_RVPF) rv.pl[rv.n++] = pl;
        } else {   // S:506 break; with FUSE the seed fit of S:513-514 (same alive set, same LPR height) is already there
          if (fuse_ok) {
            if (nsel[1] > 0) { pl = s_plane2; have_plane = true; }
            seed_done = true;
          }
          break;
        }
      }
    }
    // 2. R-GPF (S:513-543)
    if (!seed_done) {
      const double lpr = select_lpr();
      c[2] = lpr;
      fit_pass(0, false, float_ru(lpr + ap.th_seeds), 0.f, pl, c);
      if (nsel[0] > 0) { pl = s_plane; have_plane = true; }
    }
    int n_ground = 0;
    for (int it = 0; it < ap.num_iter - 1; ++it) {
      if (!have_plane) break;
      const Plane cls = pl;
      const double cc[3] = {pl.mean[0], pl.mean[1], pl.mean[2]};
      fit_pass(1, false, 0.f, 0.f, cls, cc);
      if (nsel[0] > 0) pl = s_plane;
    }
    // last iteration (S:528-542): split by the current plane, then refit on the ground part
    if (have_plane) {
      const Plane cls = pl;
      {
        const double cc[3] = {pl.mean[0], pl.mean[1], pl.mean[2]};
        fit_pass(1, false, 0.f, 0.f, cls, cc);
        n_ground = nsel[0];
        if (n_ground > 0) pl = s_plane;
      }
      PlaneF pf;
      pf.n0 = (float) cls.normal[0]; pf.n1 = (float) cls.normal[1]; pf.n2 = (float) cls.normal[2]; pf.d = (float) cls.d;
      int g_run = 0, ng_run = 0, tile = 0;
      for (int base = 0; base < n; base += NT, ++tile) {
        const int i = base + tid;
        const bool valid = i < n;
        bool is_g = false;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid) {
          p = P[i];
          int rmk = 0;   // the R-VPF iteration that removed the point (S:495-504), 0 = still alive
          for (int k = 0; k < rv.n; ++k) if (rmk == 0 && fabs(point_plane_distance(rv.pl[k], p.x, p.y, p.z)) < ap.th_dist_v) rmk = k + 1;   // S:499
          if (rmk == 0) {
            int fl = dist_filter(pf, thf, p.x, p.y, p.z);
            if (fl < 0) fl = (point_plane_distance(cls, p.x, p.y, p.z) < ap.th_dist) ? 1 : 0;
            is_g = fl != 0;
          }
          if (wq.labels) wq.labels[start + i] = is_g ? PW_LABEL_GROUND : (unsigned char) rmk;   // (PW_LABEL_REJECT == 0)
        }
        const unsigned bg = __ballot_sync(0xffffffffu, valid && is_g);
        const unsigned bn = __ballot_sync(0xffffffffu, valid && !is_g);
        const int buf = tile & 1;
        if (lane == 0) { s_wcnt[buf][w][0] = __popc(bg); s_wcnt[buf][w][1] = __popc(bn); }
        __syncthreads();
        int pg = 0, pn = 0, tg = 0, tn = 0;
#pragma unroll
        for (int q = 0; q < NW; ++q) {
          const int x = s_wcnt[buf][q][0], y = s_wcnt[buf][q][1];
          if (q < w) { pg += x; pn += y; }
          tg += x; tn += y;
        }
        if (valid) {
          const int idx = __float_as_int(p.w);
          if (is_g) out[g_run + pg + __popc(bg & lt)] = idx;
          else out[n_ground + ng_run + pn + __popc(bn & lt)] = idx;
        }
        g_run += tg;
        ng_run += tn;
      }
    } else {
      for (int i = tid; i < n; i += NT) { out[i] = __float_as_int(P[i].w); if (wq.labels) wq.labels[start + i] = PW_LABEL_REJECT; }
    }
    if (tid == 0) {
      BinFit& r = fits[(size_t) f * gs.nbs + bin];
      r.n = n; r.n_ground = n_ground; r.fitted = 1;
      r.verdict = have_plane ? 0 : PW_FIT_NO_PLANE;
#pragma unroll
      for (int k = 0; k < 3; ++k) { r.mean[k] = pl.mean[k]; r.normal[k] = pl.normal[k]; r.sv[k] = pl.sv[k]; }
      r.d = pl.d;
    }
    __syncthreads();   // s_item, s_plane*, s_n are rewritten by the next patch
  }
}

}  // namespace pwpp

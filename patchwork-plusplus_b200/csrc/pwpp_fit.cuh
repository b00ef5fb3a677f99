// pwpp_fit.cuh — per-patch plane fitting kernels (R-VPF + R-GPF), the compute-heavy stage of the path.
//
// Reference: cpp/patchworkpp/src/patchworkpp.cpp ("S:") extract_piecewiseground 467-549, extract_initial_seeds
// 77-149, estimate_plane 47-75, calc_point_to_plane_d 551-554; the per-bin sort at S:199 is not needed (see below).
//
// Design: patches are grouped by size into classes, each served by a persistent kernel that pulls self-describing
// work items (frame, bin, size, offset) from a device-side queue filled by k_bin_scan, so that every class keeps its points
// in the fastest storage they fit in and re-reads HBM never:
//     class S   n <= 64     k_fit_resident: 8 lanes x 8 points in registers, 4 patches per warp, no block barriers
//     class M   n <= 512    k_fit_warp<STAGE>: one warp per patch, patch staged once in 8 KB of shared memory
//     class L1  n <= 2048   k_fit_warp: one warp per patch, points streamed from L2, 4 loads in flight per lane
//     class L2  n <= 4096   k_fit_cta: one CTA per patch, SoA coordinates in 48 KB of shared memory
//     class L3  n <= 8192   k_fit_cta: 96 KB of shared memory
//     class X   n >  8192   k_fit_big (pwpp_fit_big.cuh): one CTA per patch streaming from L2 (dense sensors);
//                           k_fit_stream below is the one-warp-per-patch fallback (PWPP_X_KERNEL=0)
// A patch advances in "rounds": one pass over its points (seed selection or distance filter + moment accumulation in
// double) followed by ONE closed-form 3x3 eigen-solve (pwpp_math.cuh). R-GPF rounds are incremental (only points whose
// membership changed touch the double-precision sums) and stop at the exact fixpoint; zone-0 patches fuse the R-VPF fit
// with the R-GPF seed fit (FUSE, see k_fit_warp).
//
// What replaces the reference's sort: the z-sorted order is only used for (a) the count of points below the
// adaptive margin in zone 0 (S:88-96), (b) the mean of the num_lpr lowest remaining z (S:99-103) and (c) the
// seed threshold test (S:107-111). (a) and (c) are order-free predicates; (b) is a K-smallest selection, done
// here by a 32-step bisection on order-preserving integer keys with group-wide counting.
#pragma once
#include <cuda_runtime.h>

#include "pwpp_common.cuh"

namespace pwpp {

constexpr int FIT_THREADS = 256;
constexpr int CLS_S_MAX = 64, CLS_M_MAX = 512, CLS_L1_MAX = 2048, CLS_L2_MAX = 4096, CLS_L3_MAX = 8192;
constexpr int NUM_CLASSES = 6;  // S, M, L1, L2, L3, X

// device-side work queues, filled by k_bin_scan. An item describes one patch completely, so that a fit kernel needs
// a single load between claiming a queue position and touching the patch's points:
//   x = (frame << 12) | bin,  y = number of points,  (z, w) = low / high word of the patch's offset into the
//   bin-sorted point array (frame offset + bin offset)
struct WorkQueues {
  int4* items[NUM_CLASSES];
  int* count;                // [NUM_CLASSES]  number of items
  int* head;                 // [NUM_CLASSES]  next item to hand out (persistent kernels)
  // Reference-order output (pwpp_set_output_order): when non-null, every fit kernel records for each point of a fitted patch,
  // at its position in the bin-sorted array, what became of it: PW_LABEL_GROUND, PW_LABEL_REJECT (non-ground by the final
  // distance test, S:529-541) or 1..num_iter = the R-VPF iteration that removed it (S:495-504). k_order sorts by it.
  unsigned char* labels;
};
#define PW_LABEL_GROUND 255
#define PW_LABEL_REJECT 0
__device__ __forceinline__ int4 make_work_item(int frame, int bin, int n, long long start) {
  return make_int4((frame << 12) | bin, n, (int) (unsigned) (start & 0xffffffffll), (int) (start >> 32));
}
__device__ __forceinline__ long long work_item_start(const int4& w) { return ((long long) w.w << 32) | (long long) (unsigned) w.z; }
// Pull the lines of a patch that will be processed next towards L2 (fire and forget): lanes stride over 128-byte lines.
__device__ __forceinline__ void prefetch_patch_l2(const float4* P, int n, int lane, int nlanes) {
  const int lines = (n + 7) >> 3;
  for (int l = lane; l < lines; l += nlanes) prefetch_l2(P + (size_t) l * 8);
}

__device__ __forceinline__ unsigned order_key(float z) {
  const unsigned u = __float_as_uint(z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(unsigned k) {
  const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

// k-th smallest (1-based `target`) of a set of order keys all lying in [kmin, kmax]; count_less(c) must return the
// number of set members with key < c (uniform across the cooperating lanes). Bits above the highest bit in which
// kmin and kmax differ are shared by every key, so the bisection starts below them (z values of one patch
// typically share sign, exponent and a few mantissa bits: ~18 steps instead of 32).
template <typename F>
__device__ __forceinline__ unsigned kth_key(unsigned kmin, unsigned kmax, int target, F count_less) {
  const unsigned diff = kmin ^ kmax;
  if (diff == 0u) return kmin;
  const int top = 31 - __clz(diff);
  unsigned ans = (top == 31) ? 0u : (kmin & ~((2u << top) - 1u));
  for (int bit = top; bit >= 0; --bit) {
    const unsigned cand = ans | (1u << bit);
    if (count_less(cand) < target) ans = cand;
  }
  return ans;
}

// ---- group-wide reductions -------------------------------------------------------------------------
// G = 8 / 16: four / two independent groups per warp (butterfly inside 8- / 16-lane segments); G = 32: one warp.
template <int G>
struct GroupOps;

template <>
struct GroupOps<8> {
  __device__ static __forceinline__ unsigned min_u(unsigned v) {
    v = min(v, __shfl_xor_sync(0xffffffffu, v, 4)); v = min(v, __shfl_xor_sync(0xffffffffu, v, 2)); v = min(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return v;
  }
  __device__ static __forceinline__ unsigned max_u(unsigned v) {
    v = max(v, __shfl_xor_sync(0xffffffffu, v, 4)); v = max(v, __shfl_xor_sync(0xffffffffu, v, 2)); v = max(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return v;
  }
  __device__ static __forceinline__ int sum_i(int v, void*) {
    v += __shfl_xor_sync(0xffffffffu, v, 4); v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
  }
  __device__ static __forceinline__ double sum_d(double v, void*) {
    v += __shfl_xor_sync(0xffffffffu, v, 4); v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
  }
};
template <>
struct GroupOps<16> {   // two independent groups per warp (butterfly inside 16-lane segments)
  __device__ static __forceinline__ unsigned min_u(unsigned v) {
    v = min(v, __shfl_xor_sync(0xffffffffu, v, 8)); v = min(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = min(v, __shfl_xor_sync(0xffffffffu, v, 2)); v = min(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return v;
  }
  __device__ static __forceinline__ unsigned max_u(unsigned v) {
    v = max(v, __shfl_xor_sync(0xffffffffu, v, 8)); v = max(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = max(v, __shfl_xor_sync(0xffffffffu, v, 2)); v = max(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return v;
  }
  __device__ static __forceinline__ int sum_i(int v, void*) {
    v += __shfl_xor_sync(0xffffffffu, v, 8); v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
  }
  __device__ static __forceinline__ double sum_d(double v, void*) {
    v += __shfl_xor_sync(0xffffffffu, v, 8); v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
  }
};
template <>
struct GroupOps<32> {
  __device__ static __forceinline__ unsigned min_u(unsigned v) { return __reduce_min_sync(0xffffffffu, v); }
  __device__ static __forceinline__ unsigned max_u(unsigned v) { return __reduce_max_sync(0xffffffffu, v); }
  __device__ static __forceinline__ int sum_i(int v, void*) { return __reduce_add_sync(0xffffffffu, v); }
  __device__ static __forceinline__ double sum_d(double v, void*) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  }
};
// ---- transposed moment reductions ------------------------------------------------------------------
// Sum of N doubles per lane over an aligned group of D*2 lanes as a reduce-scatter: at the step of distance d a lane keeps
// one half of its values (the lower half if lane bit d is clear, else the upper half) and receives the partner's partial
// of that half, so the values exchanged halve with every step (N = 9: 12 shuffles, 18: 20) instead of N per step. Once
// one value is left the remaining steps are plain butterflies. Every partial is the sum the xor butterfly forms at the
// same step (lane + lane ^ d, and IEEE addition commutes), so each total is bit-identical to warp_sum / GroupOps::sum_d,
// in every lane that holds it. Afterwards quantity q is in slot rs_slot(N, D, q) of lane rs_lane(N, D, q) of the group.
// (not recursive, so that the compiler folds them at the unrolled call sites)
__host__ __device__ __forceinline__ constexpr int rs_lane(int n, int d, int q) {
  int l = 0;
  for (; d > 0 && n > 1; d >>= 1) { const int h = (n + 1) / 2; if (q >= h) { l |= d; q -= h; } n = h; }
  return l;
}
__host__ __device__ __forceinline__ constexpr int rs_slot(int n, int d, int q) {
  for (; d > 0 && n > 1; d >>= 1) { const int h = (n + 1) / 2; if (q >= h) q -= h; n = h; }
  return q;
}
template <int N, int D, int CAP>
__device__ __forceinline__ void reduce_scatter(double (&v)[CAP], int lane) {
  if constexpr (D > 0) {
    if constexpr (N == 1) {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], D);
      reduce_scatter<1, D / 2>(v, lane);
    } else {
      constexpr int H = (N + 1) / 2;
      const bool up = (lane & D) != 0;
#pragma unroll
      for (int k = 0; k < H; ++k) {
        const double lo = v[k], hi = (k + H < N) ? v[(k + H < N) ? k + H : 0] : 0.0;
        const double r = __shfl_xor_sync(0xffffffffu, up ? lo : hi, D);
        v[k] = (up ? hi : lo) + r;
      }
      reduce_scatter<H, D / 2>(v, lane);
    }
  }
}
// Group-wide sums of v[0..N) in every lane of the group of G lanes: reduce-scatter, then one shuffle per quantity.
template <int N, int G>
__device__ __forceinline__ void group_sum_all(double (&v)[N], int lane) {
  reduce_scatter<N, G / 2>(v, lane);
  double r[N];
#pragma unroll
  for (int q = 0; q < N; ++q) r[q] = __shfl_sync(0xffffffffu, v[rs_slot(N, G / 2, q)], rs_lane(N, G / 2, q), G);
#pragma unroll
  for (int q = 0; q < N; ++q) v[q] = r[q];
}
// the 9 moment sums of m over the group (m.n is left alone)
template <int G>
__device__ __forceinline__ void group_sum_moments(Moments& m, int lane) {
  double v[9] = {m.s1[0], m.s1[1], m.s1[2], m.s2[0], m.s2[1], m.s2[2], m.s2[3], m.s2[4], m.s2[5]};
  group_sum_all<9, G>(v, lane);
#pragma unroll
  for (int q = 0; q < 3; ++q) m.s1[q] = v[q];
#pragma unroll
  for (int q = 0; q < 6; ++q) m.s2[q] = v[3 + q];
}

enum FitState { ST_RVPF = 0, ST_SEED = 1, ST_GPF = 2, ST_FINAL = 3, ST_DONE = 4 };

// The register-resident fit kernel (classes S and M). G lanes cooperate on one patch, K points per lane; a warp
// holds 32/G patches and is completely independent of the other warps of its CTA (no block barriers): it pulls its
// own work items from the queue and every lane of a group evaluates the 3x3 eigen-problem of its patch redundantly
// (the butterfly reductions leave bit-identical moments in all lanes of the group).
// Point j of a patch lives in lane (j % G) of the group at register slot (j / G).
template <int G, int K, int CLS, int MINB>
__global__ void __launch_bounds__(FIT_THREADS, MINB) k_fit_resident(const float4* __restrict__ sorted, FrameTable ft, const StreamState* __restrict__ states,
                                                                 const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps, int nbp, const int* __restrict__ bin_off, WorkQueues wq,
                                                                 int* __restrict__ part, BinFit* __restrict__ fits) {
  static_assert(G == 8 || G == 16 || G == 32, "group is a warp, half a warp or a quarter warp");
  constexpr int NGW = 32 / G;                  // patches per warp
  const int lane = threadIdx.x & 31;
  const int gw = lane / G;                     // group inside the warp
  const int gl = lane % G;                     // lane inside the group
  typedef GroupOps<G> Ops;

  const int count = wq.count[CLS];
  int base = 0;
  if (lane == 0) base = atomicAdd(&wq.head[CLS], NGW);
  base = __shfl_sync(0xffffffffu, base, 0);
  for (;;) {
    if (base >= count) return;
    // claim the next NGW patches now: the atomic's round trip overlaps the processing of the current ones
    int next_raw = 0;
    if (lane == 0) next_raw = atomicAdd(&wq.head[CLS], NGW);
    const bool have = (base + gw) < count;
    int n = 0, bin = 0, f = 0;
    const float4* P = nullptr;
    int* out = nullptr;
    if (have) {
      const int4 wi = wq.items[CLS][base + gw];
      f = wi.x >> 12; bin = wi.x & 0xfff;
      n = wi.y;
      const long long start = work_item_start(wi);
      P = sorted + start;
      out = part + start;
    }
    const int set = ft.pset[f];                  // the parameter set of this group's frame
    const Geometry& g = gs.g[set];
    const AlgoParams& ap = aps.a[set];
    // ---- load the patches of this warp into registers ----
    float px[K], py[K], pz[K];
    unsigned vmask = 0;                        // bit k: slot k holds a point
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int j = k * G + gl;
      px[k] = 0.f; py[k] = 0.f; pz[k] = 0.f;
      if (j < n) { const float4 p = P[j]; px[k] = p.x; py[k] = p.y; pz[k] = p.z; vmask |= 1u << k; }
    }
    // slots in use by ANY patch of this warp (warp-uniform): loops over k stop there
    int kmax = (n + G - 1) / G;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, kmax, o); kmax = t > kmax ? t : kmax; }
    if (kmax > K) kmax = K;
    unsigned amask = vmask;                    // alive = not removed by R-VPF (S:495-504)
    const int zone = (bin >= g.bin_base[3]) ? 3 : (bin >= g.bin_base[2]) ? 2 : (bin >= g.bin_base[1]) ? 1 : 0;
    const bool zone0 = (zone == 0);
    // S:90; (double) z < margin  <=>  z < margin_f (float_ru), folded with the zone-0 condition
    const float margin_f = (have && zone0) ? float_ru(ap.adaptive_seed_selection_margin * states[ft.stream[f]].sensor_height) : -INFINITY;
    double c0x = 0.0, c0y = 0.0;               // first point: reference point of the shifted moments of the seed fits
    if (have) { const float4 p = P[0]; c0x = (double) p.x; c0y = (double) p.y; }

    int state = have ? ((ap.enable_RVPF && zone0) ? ST_RVPF : ST_SEED) : ST_DONE;  // zone != 0: the R-VPF fit is dead code (see k_fit_stream)
    int rvpf_it = 0, gpf_it = 0, n_ground = 0;
    bool have_plane = false;
    Plane pl;
    pl.d = 0.0;
#pragma unroll
    for (int q = 0; q < 3; ++q) { pl.mean[q] = 0.0; pl.normal[q] = 0.0; pl.sv[q] = 0.0; }
    unsigned gmask = 0, prev_sel = 0;
    bool have_prev = false;   // prev_sel is the set the current plane was fitted to (a SEED / GPF round, not R-VPF)

    // ---- rounds: one pass over the points + one plane fit each ----
    while (__any_sync(0xffffffffu, state != ST_DONE)) {
      const bool active = state != ST_DONE;
      const bool seed_round = active && (state == ST_RVPF || state == ST_SEED);
      const bool seed_round_was_rvpf = (state == ST_RVPF);
      double c[3] = {pl.mean[0], pl.mean[1], pl.mean[2]};
      float zthr = 0.f;   // float_ru of the seed threshold
      // (1) LPR selection for seed rounds: 32-step bisection on order-preserving keys with group-wide counting
      if (__any_sync(0xffffffffu, seed_round)) {
        unsigned smask = 0;  // candidates: alive and not below the zone-0 margin (S:88-96)
        unsigned keys[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
          keys[k] = order_key(pz[k]);
          const bool ok = seed_round && ((amask >> k) & 1u) && !(pz[k] < margin_f);
          smask |= ok ? (1u << k) : 0u;
        }
        const int nvalid = Ops::sum_i(__popc(smask), nullptr);
        const int target = nvalid < ap.num_lpr ? nvalid : ap.num_lpr;
        unsigned kmn = 0xffffffffu, kmx = 0u;
#pragma unroll
        for (int k = 0; k < K; ++k) if ((smask >> k) & 1u) { kmn = min(kmn, keys[k]); kmx = max(kmx, keys[k]); }
        kmn = Ops::min_u(kmn); kmx = Ops::max_u(kmx);
        // the groups of a warp bisect together: use the widest range among them so that the loop is warp-uniform
        unsigned ans = 0;
        {
          unsigned diff = (nvalid > 0) ? (kmn ^ kmx) : 0u;
          diff = __reduce_or_sync(0xffffffffu, diff);
          const int top = diff ? (31 - __clz(diff)) : -1;
          ans = (nvalid > 0) ? ((top >= 31 || top < 0) ? (top < 0 ? kmn : 0u) : (kmn & ~((2u << top) - 1u))) : 0u;
          for (int bit = top; bit >= 0; --bit) {
            const unsigned cand = ans | (1u << bit);
            int cnt = 0;
#pragma unroll
            for (int k = 0; k < K; ++k) { if (k >= kmax) break; cnt += (((smask >> k) & 1u) && keys[k] < cand) ? 1 : 0; }
            cnt = Ops::sum_i(cnt, nullptr);
            if (cnt < target) ans = cand;
          }
        }
        // ans = the target-th smallest key; mean of the target lowest z (S:99-103)
        double part_sum = 0.0;
        int c_lt = 0;
#pragma unroll
        for (int k = 0; k < K; ++k)
          if (((smask >> k) & 1u) && keys[k] < ans) { part_sum += (double) pz[k]; ++c_lt; }
        part_sum = Ops::sum_d(part_sum, nullptr);
        c_lt = Ops::sum_i(c_lt, nullptr);
        double lpr = 0.0;
        if (target > 0) lpr = (part_sum + (double) (target - c_lt) * (double) key_to_float(ans)) / (double) target;
        if (seed_round) {
          zthr = float_ru(lpr + (state == ST_RVPF ? ap.th_seeds_v : ap.th_seeds));
          c[0] = c0x; c[1] = c0y; c[2] = lpr;
        }
      }
      // (2) predicate + moments
      Moments m;
      m.n = 0;
#pragma unroll
      for (int q = 0; q < 3; ++q) m.s1[q] = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) m.s2[q] = 0.0;
      unsigned sel = 0;
      if (active) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
          if (k >= kmax) break;
          bool in = (amask >> k) & 1u;
          if (seed_round) in = in && (pz[k] < zthr);                                                   // S:108 / S:145
          else in = in && have_plane && (point_plane_distance(pl, px[k], py[k], pz[k]) < ap.th_dist);  // S:525 / S:529
          if (in) {
            sel |= 1u << k;
            const double dx = (double) px[k] - c[0], dy = (double) py[k] - c[1], dz = (double) pz[k] - c[2];
            m.s1[0] += dx; m.s1[1] += dy; m.s1[2] += dz;
            m.s2[0] += dx * dx; m.s2[1] += dx * dy; m.s2[2] += dx * dz;
            m.s2[3] += dy * dy; m.s2[4] += dy * dz; m.s2[5] += dz * dz;
            m.n += 1;
          }
        }
      }
      group_sum_moments<G>(m, lane);
      m.n = Ops::sum_i(m.n, nullptr);
      // every lane of the warp takes part in this reduction (the groups of a warp are in different states)
      const bool set_unchanged = Ops::sum_i((active && sel != prev_sel) ? 1 : 0, nullptr) == 0;
      // (3) plane of the selected set; an empty set keeps the previous plane (S:49)
      if (active && m.n > 0) { plane_from_moments(m, c, pl); have_plane = true; }
      // (4) state transition
      if (state == ST_RVPF) {
        if (have_plane && pl.normal[2] < ap.uprightness_thr) {  // S:489: remove the vertical structure, iterate
#pragma unroll
          for (int k = 0; k < K; ++k)
            if (((amask >> k) & 1u) && fabs(point_plane_distance(pl, px[k], py[k], pz[k])) < ap.th_dist_v) {   // S:499
              amask &= ~(1u << k);
              if (wq.labels) wq.labels[(P - sorted) + k * G + gl] = (unsigned char) (rvpf_it + 1);
            }
          ++rvpf_it;
          if (rvpf_it >= ap.num_iter) state = ST_SEED;
        } else state = ST_SEED;  // S:506 break
      } else if (state == ST_SEED) {
        state = (ap.num_iter > 1) ? ST_GPF : ST_FINAL;
        gpf_it = 0;
      } else if (state == ST_GPF) {
        ++gpf_it;
        if (gpf_it >= ap.num_iter - 1) state = ST_FINAL;
        // fixpoint of S:516-543: the set selected by the current plane equals the set that plane was fitted to,
        // so every later iteration selects it again and refits the same plane
        if (set_unchanged && have_prev) { gmask = sel; n_ground = m.n; state = ST_DONE; }
      } else if (state == ST_FINAL) {
        gmask = sel;
        n_ground = m.n;
        state = ST_DONE;
      }
      if (active) { have_prev = !seed_round_was_rvpf; prev_sel = sel; }
    }

    // ---- stable partition: ground indices ascending, then non-ground indices ascending ----
    {
      // every lane runs the ballots (lanes of absent patches hold no valid slot); only valid slots store
      const unsigned seg_shift = (G < 32) ? (unsigned) ((lane / G) * G) : 0u;
      const unsigned seg_mask = (G < 32) ? ((1u << (G & 31)) - 1u) : 0xffffffffu;
      const unsigned lt = ((G < 32) ? ((1u << (lane % G)) - 1u) : lanemask_lt());
      int g_run = 0, ng_run = 0;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        if (k >= kmax) break;
        const bool v = (vmask >> k) & 1u, isg = (gmask >> k) & 1u;
        const unsigned bg = (__ballot_sync(0xffffffffu, v && isg) >> seg_shift) & seg_mask;
        const unsigned bn = (__ballot_sync(0xffffffffu, v && !isg) >> seg_shift) & seg_mask;
        if (v) {
          const int j = k * G + gl;
          const int idx = __float_as_int(P[j].w);
          if (isg) out[g_run + __popc(bg & lt)] = idx;
          else out[n_ground + ng_run + __popc(bn & lt)] = idx;
          if (wq.labels && (isg || ((amask >> k) & 1u))) wq.labels[(P - sorted) + j] = isg ? PW_LABEL_GROUND : PW_LABEL_REJECT;
        }
        g_run += __popc(bg);
        ng_run += __popc(bn);
      }
      if (have && gl == 0) {
        BinFit& r = fits[(size_t) f * gs.nbs + bin];
        r.n = n; r.n_ground = n_ground; r.fitted = 1;
        r.verdict = have_plane ? 0 : PW_FIT_NO_PLANE;
#pragma unroll
        for (int q = 0; q < 3; ++q) { r.mean[q] = pl.mean[q]; r.normal[q] = pl.normal[q]; r.sv[q] = pl.sv[q]; }
        r.d = pl.d;
      }
    }
    __syncwarp();
    base = __shfl_sync(0xffffffffu, next_raw, 0);
  }
}

struct PlaneF { float n0, n1, n2, d; };

// +1: surely below th_dist, 0: surely not, -1: inside the fp32 error bound (decide in double)
__device__ __forceinline__ int dist_filter(const PlaneF& pf, float th, float x, float y, float z) {
  const float sf = fmaf(pf.n0, x, fmaf(pf.n1, y, fmaf(pf.n2, z, pf.d)));
  // |sf - exact| <= 3e-7 * (|x|+|y|+|z|+|d|) (|n_i| <= 1: float coefficients + three fma roundings); 3x margin
  const float bound = 1e-6f * (fabsf(x) + fabsf(y) + fabsf(z) + fabsf(pf.d) + 1.0f);
  const float diff = sf - th;
  return (fabsf(diff) > bound) ? (diff < 0.f ? 1 : 0) : -1;
}

// ---------------------------------------------------------------------------------------------------
// k_fit_cta: one CTA per patch, coordinates staged once in shared memory (SoA), CAP points at most.
// Warp w owns the contiguous index range [w*chunk, (w+1)*chunk); a thread's slot `it` is point
// w*chunk + it*32 + lane, so shared-memory accesses are conflict free and the final stable partition needs one
// cross-warp prefix. The LPR selection is two-level: the num_lpr-th smallest of the 256 per-thread minima bounds
// the num_lpr-th smallest point from above, so only the few points not above that bound are gathered and
// selected exactly by one warp.
// PLS (PWPP_L2_PLS): the current plane lives in shared memory (s_plane) instead of 20 registers per thread — warp 0 rewrites it
// in place between the two barriers of a round, when no other warp reads it — so that the fused kernel fits the 64-register
// budget of 4 CTAs per SM with far fewer spills.
template <int CAP, int CLS, int MINB, int NW, bool FUSE = false, bool PLS = false>
__global__ void __launch_bounds__(NW * 32, MINB) k_fit_cta(const float4* __restrict__ sorted, FrameTable ft, const StreamState* __restrict__ states,
                                                                                const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps, int nbp, const int* __restrict__ bin_off, WorkQueues wq,
                                                                                int* __restrict__ part, BinFit* __restrict__ fits) {
  constexpr int NT = NW * 32;                // NW warps per patch (8 or 16)
  static_assert(NW == 8 || NW == 16, "warp 0 keeps NW minima per lane and splits a patch into NW contiguous chunks");
  static_assert(CAP / NT <= 32, "slot masks are 32-bit");
  constexpr int CCAP = 512;
  PW_DYN_SHARED(float, s_pts);
  float* sx = s_pts;
  float* sy = sx + CAP;
  float* sz = sy + CAP;
  __shared__ double s_part[2][NW][9];   // per-warp partial moments, double-buffered by round parity
  __shared__ double s_parti[FUSE ? 2 : 1][FUSE ? NW : 1][9];   // FUSE: the inner (R-GPF seed) set of a fused round
  __shared__ int s_pcnt[2][NW], s_pchg[2][NW];
  __shared__ Plane s_plane2;            // FUSE: the R-GPF seed plane of a fused round
  __shared__ int s_mni, s_taken;
  __shared__ int s_cnt[NW][2];
  __shared__ unsigned s_min[NT];
  __shared__ unsigned s_cand[CCAP];
  __shared__ double s_lpr;
  __shared__ double s_fb[NW];
  __shared__ unsigned s_T;
  __shared__ int s_ccount, s_mn, s_fix, s_refit;
  __shared__ int4 s_item;
  __shared__ Plane s_plane;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int count = wq.count[CLS];
  const int4 no_item = make_int4(-1, 0, 0, 0);

  // Queue protocol: the last warp claims one patch AHEAD — the atomic at the top of a patch, the descriptor load after
  // the staging loads, an L2 prefetch of that patch's points while warp 0 solves the first plane (when the other
  // warps idle anyway) — and publishes the descriptor through s_item at the end of the patch; x < 0 = queue drained.
  constexpr int LOOK_W = NW - 1, LOOK_TID = LOOK_W * 32;
  if (tid == 0) {
    const int t = atomicAdd(&wq.head[CLS], 1);
    s_item = t < count ? wq.items[CLS][t] : no_item;
  }
  __syncthreads();
  for (;;) {
    const int4 cur = s_item;
    if (cur.x < 0) return;
    int next_raw = 0;
    if (tid == LOOK_TID) next_raw = atomicAdd(&wq.head[CLS], 1);
    const int f = cur.x >> 12, bin = cur.x & 0xfff, n = cur.y;
    const int set = ft.pset[f];                  // the frame's parameter set
    const Geometry& g = gs.g[set];
    const AlgoParams& ap = aps.a[set];
    const float thf = (float) ap.th_dist;
    const long long start = work_item_start(cur);
    const float4* P = sorted + start;
    int* out = part + start;
    const int chunk = (((n + NW - 1) / NW) + 31) & ~31;   // points per warp, multiple of 32
    const int nit = chunk >> 5;                      // slots per thread actually used (<= ITERS)
    const int jbase = w * chunk + lane;
    unsigned vmask = 0;
#pragma unroll 4   // (eight staging loads in flight for the L3 kernel: no difference)
    for (int it = 0; it < nit; ++it) {
      const int j = jbase + it * 32;
      if (j < n) { const float4 p = P[j]; sx[j] = p.x; sy[j] = p.y; sz[j] = p.z; vmask |= 1u << it; }
    }
    int4 nxt = no_item;   // next patch (meaningful in the look-ahead warp)
    if (w == LOOK_W) {
      const int t = __shfl_sync(0xffffffffu, next_raw, 0);
      if (t < count) nxt = wq.items[CLS][t];
    }
    unsigned amask = vmask;
    const int zone = (bin >= g.bin_base[3]) ? 3 : (bin >= g.bin_base[2]) ? 2 : (bin >= g.bin_base[1]) ? 1 : 0;
    const bool zone0 = (zone == 0);
    // S:90; (double) z < margin  <=>  z < margin_f (float_ru), folded with the zone-0 condition
    const float margin_f = zone0 ? float_ru(ap.adaptive_seed_selection_margin * states[ft.stream[f]].sensor_height) : -INFINITY;
    const float4 first = P[0];
    const double c0x = (double) first.x, c0y = (double) first.y;

    int state = (ap.enable_RVPF && zone0) ? ST_RVPF : ST_SEED;
    int rvpf_it = 0, gpf_it = 0, n_ground = 0;
    bool have_plane = false;
    Plane pl_reg;
    Plane& pl = PLS ? s_plane : pl_reg;   // PLS: nobody depends on the plane before the first barrier of the first (seed) round
    if (!PLS || tid == 0) {
      pl.d = 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) { pl.mean[q] = 0.0; pl.normal[q] = 0.0; pl.sv[q] = 0.0; }
    }
    unsigned gmask = 0, member = 0;
    int round = 0;
    double c_lpr = 0.0;
    Moments tot;   // running sums of the R-GPF phase (meaningful in warp 0)
    tot.n = 0;
#pragma unroll
    for (int q = 0; q < 3; ++q) tot.s1[q] = 0.0;
#pragma unroll
    for (int q = 0; q < 6; ++q) tot.s2[q] = 0.0;

    // FUSE: see k_fit_warp — an R-VPF round also accumulates the R-GPF seed set (same LPR height while nothing has been
    // removed in this round) and warp 0 solves both planes in its two halves; when the R-VPF plane is upright the
    // separate ST_SEED round (selection, pass, four barriers) is skipped.
    const bool fuse_ok = FUSE && (ap.th_seeds <= ap.th_seeds_v);
    while (state != ST_DONE) {   // state is uniform across the CTA
      const bool seed_round = (state == ST_RVPF || state == ST_SEED);
      const bool fused = fuse_ok && state == ST_RVPF;
      double c[3] = {pl.mean[0], pl.mean[1], pl.mean[2]};
      float zthr = 0.f, zin = 0.f;   // float_ru of the seed thresholds
      if (seed_round) {
        // ---- LPR: mean of the num_lpr lowest z among the alive points not below the zone-0 margin (S:88-103) ----
        unsigned smask = 0, kmin = 0xffffffffu;
        int nv = 0;
        for (int it = 0; it < nit; ++it) {
          if (!((amask >> it) & 1u)) continue;
          const float z = sz[jbase + it * 32];
          if (z < margin_f) continue;
          smask |= 1u << it;
          const unsigned key = order_key(z);
          kmin = key < kmin ? key : kmin;
          ++nv;
        }
        s_min[tid] = kmin;
        nv = __reduce_add_sync(0xffffffffu, nv);
        if (lane == 0) s_cnt[w][0] = nv;
        if (tid == 0) s_ccount = 0;
        __syncthreads();
        int nvalid = 0;
#pragma unroll
        for (int q = 0; q < NW; ++q) nvalid += s_cnt[q][0];
        const int target = nvalid < ap.num_lpr ? nvalid : ap.num_lpr;
        if (w == 0) {
          unsigned mk[NW];
          int have = 0;
#pragma unroll
          for (int q = 0; q < NW; ++q) { mk[q] = s_min[lane * NW + q]; have += mk[q] != 0xffffffffu; }
          have = __reduce_add_sync(0xffffffffu, have);
          unsigned ans = 0xffffffffu;   // fewer candidate-holding threads than target: keep everything
          if (target > 0 && have >= target) {
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
        for (int it = 0; it < nit; ++it) {
          if (!((smask >> it) & 1u)) continue;
          const unsigned key = order_key(sz[jbase + it * 32]);
          if (key <= T) { const int pos = atomicAdd(&s_ccount, 1); if (pos < CCAP) s_cand[pos] = key; }
        }
        __syncthreads();
        const int cc = s_ccount;
        if (cc <= CCAP) {
          if (w == 0) {   // exact selection among the gathered candidates
            unsigned ck[CCAP / 32];
            unsigned kmn = 0xffffffffu, kmx = 0u;
            const int nq = (cc + 31) >> 5;
#pragma unroll
            for (int q = 0; q < CCAP / 32; ++q) {
              const int i = lane + 32 * q;
              ck[q] = i < cc ? s_cand[i] : 0xffffffffu;
              if (i < cc) { kmn = min(kmn, ck[q]); kmx = max(kmx, ck[q]); }
            }
            kmn = __reduce_min_sync(0xffffffffu, kmn);
            kmx = __reduce_max_sync(0xffffffffu, kmx);
            const unsigned ans = kth_key(kmn, kmx, target, [&](unsigned cand) {
              int cnt = 0;
#pragma unroll
              for (int q = 0; q < CCAP / 32; ++q) { if (q >= nq) break; cnt += ck[q] < cand; }
              return __reduce_add_sync(0xffffffffu, cnt);
            });
            double ps = 0.0;
            int c_lt = 0;
#pragma unroll
            for (int q = 0; q < CCAP / 32; ++q) if (ck[q] < ans) { ps += (double) key_to_float(ck[q]); ++c_lt; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
            c_lt = __reduce_add_sync(0xffffffffu, c_lt);
            if (lane == 0) s_lpr = target > 0 ? (ps + (double) (target - c_lt) * (double) key_to_float(ans)) / (double) target : 0.0;
          }
          __syncthreads();
        } else {
          // many ties at the bound (e.g. a perfectly flat synthetic plane): CTA-wide bisection over all candidates
          unsigned ans = 0;
          for (int bit = 31; bit >= 0; --bit) {
            const unsigned cand = ans | (1u << bit);
            int cnt = 0;
            for (int it = 0; it < nit; ++it) if (((smask >> it) & 1u) && order_key(sz[jbase + it * 32]) < cand) ++cnt;
            cnt = __reduce_add_sync(0xffffffffu, cnt);
            if (lane == 0) s_cnt[w][1] = cnt;
            __syncthreads();
            int tot = 0;
#pragma unroll
            for (int q = 0; q < NW; ++q) tot += s_cnt[q][1];
            __syncthreads();
            if (tot < target) ans = cand;
          }
          double ps = 0.0;
          int c_lt = 0;
          for (int it = 0; it < nit; ++it) {
            if (!((smask >> it) & 1u)) continue;
            const float z = sz[jbase + it * 32];
            if (order_key(z) < ans) { ps += (double) z; ++c_lt; }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
          c_lt = __reduce_add_sync(0xffffffffu, c_lt);
          if (lane == 0) { s_fb[w] = ps; s_cnt[w][1] = c_lt; }
          __syncthreads();
          if (tid == 0) {
            double tps = 0.0; int tlt = 0;
            for (int q = 0; q < NW; ++q) { tps += s_fb[q]; tlt += s_cnt[q][1]; }
            s_lpr = target > 0 ? (tps + (double) (target - tlt) * (double) key_to_float(ans)) / (double) target : 0.0;
          }
          __syncthreads();
        }
        const double lpr = s_lpr;
        zthr = float_ru(lpr + (state == ST_RVPF ? ap.th_seeds_v : ap.th_seeds));
        zin = float_ru(lpr + ap.th_seeds);
        c[0] = c0x; c[1] = c0y; c[2] = lpr;
      }
      // ---- predicate + moments ----
      // Seed rounds accumulate their whole set. R-GPF rounds are incremental (see k_fit_warp): every fit of the
      // R-GPF phase shares the reference point c = (first x, first y, lpr), a round adds (+) / removes (-) only
      // the points whose membership changed, warp 0 keeps the running sums, and a round without any change is the
      // fixpoint of S:516-543.
      const bool incr = !seed_round;
      if (incr) { c[0] = c0x; c[1] = c0y; c[2] = c_lpr; }
      else if (state == ST_SEED || (FUSE && fused)) c_lpr = c[2];
      PlaneF pf;
      pf.n0 = (float) pl.normal[0]; pf.n1 = (float) pl.normal[1]; pf.n2 = (float) pl.normal[2]; pf.d = (float) pl.d;
      double a[9], bi[FUSE ? 9 : 1];
#pragma unroll
      for (int q = 0; q < 9; ++q) a[q] = 0.0;
#pragma unroll
      for (int q = 0; q < (FUSE ? 9 : 1); ++q) bi[q] = 0.0;
      int mn = 0, nchg = 0, mni = 0;
      unsigned sel = 0, seli = 0;
      for (int it = 0; it < nit; ++it) {
        if (!((amask >> it) & 1u)) continue;
        const int j = jbase + it * 32;
        const float x = sx[j], y = sy[j], z = sz[j];
        bool in;
        if (seed_round) in = (z < zthr);                                                     // S:108 / S:145
        else {
          int fl = have_plane ? dist_filter(pf, thf, x, y, z) : 0;
          if (fl < 0) fl = (point_plane_distance(pl, x, y, z) < ap.th_dist) ? 1 : 0;         // S:525 / S:529, exact
          in = fl != 0;
        }
        if (in) sel |= 1u << it;
        double wgt = in ? 1.0 : 0.0;
        if (incr) {
          const bool was = (member >> it) & 1u;
          if (was == in) continue;
          wgt = in ? 1.0 : -1.0;
          ++nchg;
        } else if (!in) continue;
        const double dx = (double) x - c[0], dy = (double) y - c[1], dz = (double) z - c[2];
        const double wx = dx * wgt, wy = dy * wgt, wz = dz * wgt;
        a[0] += wx; a[1] += wy; a[2] += wz;
        a[3] += wx * dx; a[4] += wx * dy; a[5] += wx * dz; a[6] += wy * dy; a[7] += wy * dz; a[8] += wz * dz;
        mn += in ? 1 : -1;
        if (FUSE && fused && (z < zin)) {   // also a seed of the R-GPF seed fit (in is true here)
          seli |= 1u << it;
          bi[0] += dx; bi[1] += dy; bi[2] += dz;
          bi[3] += dx * dx; bi[4] += dx * dy; bi[5] += dx * dz; bi[6] += dy * dy; bi[7] += dy * dz; bi[8] += dz * dz;
          ++mni;
        }
      }
      member = (FUSE && fused) ? seli : sel;   // a fused round that is not taken recomputes everything in the next round
      mn = __reduce_add_sync(0xffffffffu, mn);
      nchg = __reduce_add_sync(0xffffffffu, nchg);
      const int buf = round & 1;
      ++round;
      // warp sums by reduce-scatter: the lane that ends up holding quantity q stores it
      if (FUSE && fused) {
        double v[18];
#pragma unroll
        for (int q = 0; q < 9; ++q) { v[q] = a[q]; v[9 + q] = bi[FUSE ? q : 0]; }
        reduce_scatter<18, 16>(v, lane);
#pragma unroll
        for (int q = 0; q < 9; ++q) {
          if (lane == rs_lane(18, 16, q)) s_part[buf][w][q] = v[rs_slot(18, 16, q)];
          if (lane == rs_lane(18, 16, 9 + q)) s_parti[FUSE ? buf : 0][FUSE ? w : 0][q] = v[rs_slot(18, 16, 9 + q)];
        }
        mni = __reduce_add_sync(0xffffffffu, mni);
        if (lane == 0) s_cnt[w][1] = mni;
      } else {
        reduce_scatter<9, 16>(a, lane);
#pragma unroll
        for (int q = 0; q < 9; ++q)
          if (lane == rs_lane(9, 16, q)) s_part[buf][w][q] = a[rs_slot(9, 16, q)];
      }
      if (lane == 0) {
        s_pcnt[buf][w] = mn;
        s_pchg[buf][w] = nchg;
      }
      __syncthreads();
      // warp 0 combines the NW partials (lane q sums quantity q over the warps in a fixed order: bit-reproducible),
      // keeps the running sums of the R-GPF phase, solves the 3x3 problem once and publishes the plane; the other
      // warps wait at the second barrier
      if (FUSE && fused) {
        if (w == 0) {
          // lanes 0..8 / 16..24 combine the moments of all seeds / the inner seeds; lanes 9 / 25 the counts
          double v = 0.0;
          int cn = 0;
          const int ql = lane & 15;
          const bool hi = lane >= 16;
          if (ql < 9) {
#pragma unroll
            for (int ww = 0; ww < NW; ++ww) v += hi ? s_parti[FUSE ? buf : 0][FUSE ? ww : 0][ql] : s_part[buf][ww][ql];
          } else if (ql == 9) {
#pragma unroll
            for (int ww = 0; ww < NW; ++ww) cn += hi ? s_cnt[ww][1] : s_pcnt[buf][ww];
          }
          Moments mv, mi;
#pragma unroll
          for (int q = 0; q < 3; ++q) { mv.s1[q] = __shfl_sync(0xffffffffu, v, q); mi.s1[q] = __shfl_sync(0xffffffffu, v, 16 + q); }
#pragma unroll
          for (int q = 0; q < 6; ++q) { mv.s2[q] = __shfl_sync(0xffffffffu, v, 3 + q); mi.s2[q] = __shfl_sync(0xffffffffu, v, 19 + q); }
          mv.n = __shfl_sync(0xffffffffu, cn, 9);
          mi.n = __shfl_sync(0xffffffffu, cn, 25);
          Moments ms = hi ? mi : mv;
          Plane mine = pl;
          if (ms.n > 0) plane_from_moments(ms, c, mine);
          const double vz = __shfl_sync(0xffffffffu, mine.normal[2], 0);
          const bool hv = have_plane || mv.n > 0;
          const bool taken = !(hv && (mv.n > 0 ? vz : pl.normal[2]) < ap.uprightness_thr);   // S:489 false -> S:506 break
          if (taken) tot = mi; else tot = mv;
          if (PLS) {   // the plane the next round uses goes straight to s_plane: the seed plane when taken and fitted, else the R-VPF plane
            const bool seed_wins = taken && mi.n > 0;
            if (lane == 0) { if (!seed_wins && mv.n > 0) s_plane = mine; s_mn = mv.n; s_refit = mv.n > 0 ? 1 : 0; s_fix = 0; s_taken = taken ? 1 : 0; }
            if (lane == 16) { if (seed_wins) s_plane = mine; s_mni = mi.n; }
          } else {
            if (lane == 0) { s_plane = mine; s_mn = mv.n; s_refit = mv.n > 0 ? 1 : 0; s_fix = 0; s_taken = taken ? 1 : 0; }
            if (lane == 16) { s_plane2 = mine; s_mni = mi.n; }
          }
        } else if (w == LOOK_W && rvpf_it == 0) {
          if (nxt.x >= 0) prefetch_patch_l2(sorted + work_item_start(nxt), nxt.y, lane, 32);
        }
      } else
      if (w == 0) {
        double v = 0.0;
        int cn = 0;
        if (lane < 9) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) v += s_part[buf][ww][lane];
        } else if (lane == 9) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) cn += s_pcnt[buf][ww];
        } else if (lane == 10) {
#pragma unroll
          for (int ww = 0; ww < NW; ++ww) cn += s_pchg[buf][ww];
        }
        Moments m;
#pragma unroll
        for (int q = 0; q < 3; ++q) m.s1[q] = __shfl_sync(0xffffffffu, v, q);
#pragma unroll
        for (int q = 0; q < 6; ++q) m.s2[q] = __shfl_sync(0xffffffffu, v, 3 + q);
        m.n = __shfl_sync(0xffffffffu, cn, 9);
        const int changed = __shfl_sync(0xffffffffu, cn, 10);
        bool refit = true;
        if (incr) {
          if (changed == 0) refit = false;   // fixpoint
          else {
#pragma unroll
            for (int q = 0; q < 3; ++q) tot.s1[q] += m.s1[q];
#pragma unroll
            for (int q = 0; q < 6; ++q) tot.s2[q] += m.s2[q];
            tot.n += m.n;
          }
        } else tot = m;
        if (refit && tot.n > 0) {
          Plane t;
          plane_from_moments(tot, c, t);
          if (lane == 0) s_plane = t;
        }
        if (lane == 0) { s_mn = tot.n; s_fix = (incr && changed == 0) ? 1 : 0; s_refit = (refit && tot.n > 0) ? 1 : 0; }
      } else if (w == LOOK_W && state == ST_SEED) {   // the R-GPF seed round: exactly once per patch
        if (nxt.x >= 0) prefetch_patch_l2(sorted + work_item_start(nxt), nxt.y, lane, 32);
      }
      __syncthreads();
      int tot_n = s_mn;
      const bool fixpoint = s_fix != 0;
      if (s_refit) { if (!PLS) pl = s_plane; have_plane = true; }   // S:49: an empty set keeps the previous plane
      // ---- state transition (same machine as k_fit_resident) ----
      if (FUSE && fused && s_taken) {   // upright R-VPF plane (S:506 break) + the seed fit of S:513-514 from the same pass
        tot_n = s_mni;
        if (tot_n > 0) { if (!PLS) pl = s_plane2; have_plane = true; }
        state = (ap.num_iter > 1) ? ST_GPF : ST_FINAL;
        gpf_it = 0;
      } else
      if (state == ST_RVPF) {
        if (have_plane && pl.normal[2] < ap.uprightness_thr) {   // S:489
          for (int it = 0; it < nit; ++it) {
            if (!((amask >> it) & 1u)) continue;
            const int j = jbase + it * 32;
            if (fabs(point_plane_distance(pl, sx[j], sy[j], sz[j])) < ap.th_dist_v) {   // S:499
              amask &= ~(1u << it);
              if (wq.labels) wq.labels[start + j] = (unsigned char) (rvpf_it + 1);
            }
          }
          ++rvpf_it;
          if (rvpf_it >= ap.num_iter) state = ST_SEED;
        } else state = ST_SEED;
      } else if (state == ST_SEED) {
        state = (ap.num_iter > 1) ? ST_GPF : ST_FINAL;
        gpf_it = 0;
      } else if (state == ST_GPF) {
        ++gpf_it;
        if (gpf_it >= ap.num_iter - 1) state = ST_FINAL;
        if (fixpoint) state = ST_DONE;
      } else {   // ST_FINAL
        state = ST_DONE;
      }
      if (state == ST_DONE) { gmask = have_plane ? member : 0u; n_ground = have_plane ? tot_n : 0; }
    }

    // ---- stable partition: ground indices ascending, then non-ground indices ascending ----
    {
      const int gw = __reduce_add_sync(0xffffffffu, __popc(gmask));
      const int nw = __reduce_add_sync(0xffffffffu, __popc(vmask & ~gmask));
      if (lane == 0) { s_cnt[w][0] = gw; s_cnt[w][1] = nw; }
      __syncthreads();
      int g_run = 0, ng_run = 0;
      for (int q = 0; q < w; ++q) { g_run += s_cnt[q][0]; ng_run += s_cnt[q][1]; }
      const unsigned lt = lanemask_lt();
      for (int it0 = 0; it0 < nit; it0 += 4) {   // four index loads in flight per thread (they come from L2, and with one in flight this load was a top stall site)
        int idxb[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int it = it0 + u; idxb[u] = (it < nit && ((vmask >> it) & 1u)) ? __float_as_int(P[jbase + it * 32].w) : 0; }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int it = it0 + u;
          if (it >= nit) break;
          const bool v = (vmask >> it) & 1u, isg = (gmask >> it) & 1u;
          const unsigned bg = __ballot_sync(0xffffffffu, v && isg);
          const unsigned bn = __ballot_sync(0xffffffffu, v && !isg);
          if (v) {
            const int idx = idxb[u];
            if (isg) out[g_run + __popc(bg & lt)] = idx;
            else out[n_ground + ng_run + __popc(bn & lt)] = idx;
            if (wq.labels && (isg || ((amask >> it) & 1u))) wq.labels[start + jbase + it * 32] = isg ? PW_LABEL_GROUND : PW_LABEL_REJECT;
          }
          g_run += __popc(bg);
          ng_run += __popc(bn);
        }
      }
      if (tid == 0) {
        BinFit& r = fits[(size_t) f * gs.nbs + bin];
        r.n = n; r.n_ground = n_ground; r.fitted = 1;
        r.verdict = have_plane ? 0 : PW_FIT_NO_PLANE;
#pragma unroll
        for (int q = 0; q < 3; ++q) { r.mean[q] = pl.mean[q]; r.normal[q] = pl.normal[q]; r.sv[q] = pl.sv[q]; }
        r.d = pl.d;
      }
      if (tid == LOOK_TID) s_item = nxt;   // every thread read the current descriptor before the barrier above
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------
// Streaming fallback (class X, patches larger than the register-resident kernels hold): one warp per patch,
// points re-read from L2 in every pass, R-VPF removals re-evaluated from the stored planes.

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) { return __reduce_add_sync(0xffffffffu, v); }

// Bitonic sort of 128 floats in shared memory by one warp (ascending).
__device__ __forceinline__ void warp_sort128(float* buf) {
  const int lane = lane_id();
  for (int k = 2; k <= 128; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int idx = lane + 32 * t;                       // 0..63: pair index
        const int i = ((idx & ~(j - 1)) << 1) | (idx & (j - 1));  // lower element of the pair
        const int l = i | j;
        const bool up = ((i & k) == 0);
        const float a = buf[i], b = buf[l];
        if ((a > b) == up) { buf[i] = b; buf[l] = a; }
      }
      __syncwarp();
    }
  }
}

// Streaming selection of the K smallest keys: candidates below the current bound are appended to a
// 128-slot shared buffer; when it could overflow it is sorted and truncated to K.
struct LprSelector {
  float* buf;   // [128]
  int m;        // valid entries
  float tau;    // current bound: the K-th smallest so far once K are known, else +inf
  int K;
  __device__ __forceinline__ void init(float* b, int k) { buf = b; m = 0; tau = INFINITY; K = k; }
  __device__ __forceinline__ void prune() {
    const int lane = lane_id();
    for (int i = m + lane; i < 128; i += 32) buf[i] = INFINITY;
    __syncwarp();
    warp_sort128(buf);
    if (m > K) m = K;
    if (m == K) tau = buf[K - 1];
    __syncwarp();
  }
  // every lane calls with its candidate (valid == false for lanes without one)
  __device__ __forceinline__ void push(bool valid, float key) {
    const bool c = valid && (key < tau);
    const unsigned bal = __ballot_sync(0xffffffffu, c);
    if (bal == 0) return;
    if (c) buf[m + __popc(bal & lanemask_lt())] = key;
    m += __popc(bal);
    __syncwarp();
    if (m > 96) prune();
  }
};

struct RvpfPlanes {
  Plane pl[MAX_RVPF];
  int n;
};

__device__ __forceinline__ bool is_alive(const RvpfPlanes& rv, double th_dist_v, float x, float y, float z) {
  bool alive = true;
  for (int k = 0; k < rv.n; ++k) alive = alive && !(fabs(point_plane_distance(rv.pl[k], x, y, z)) < th_dist_v);  // S:499
  return alive;
}

// ---------------------------------------------------------------------------------------------------
// k_fit_warp: one warp per patch, no block-level synchronisation at all.
//   STAGE = true  (class M, 65..512 points): the patch is copied once into the warp's 8 KB of shared memory and
//                 every pass reads it from there;
//   STAGE = false (classes L2 then L1, 513..8192 points): the points are streamed from L2 in every pass, four
//                 independent 128-bit loads per lane in flight (lane l reads points l, l+32, ...).
// Per point a pass must remember one bit, kept as the ballot word of its iteration in per-warp shared memory
// (alive = not removed by R-VPF, S:495-504; member = in the set the current plane was fitted to).
//
// Two things keep the per-point cost low:
//  * the point-to-plane test (S:525/529) is first evaluated in fp32 with a rigorous error bound; only points
//    whose fp32 distance lies inside the bound of th_dist are re-evaluated in double (identical decisions);
//  * the moment sums of the R-GPF iterations are INCREMENTAL: all fits of a patch share one reference point, so a
//    round only adds (+) / removes (-) the points whose membership changed w.r.t. the previous set. A round
//    without any change has reached the fixpoint of S:516-543 (same set => same plane => same next set) and the
//    remaining iterations are skipped — exactly, not approximately.
constexpr int WARP_CAP = CLS_L3_MAX;            // 8192 points -> 256 iterations
constexpr int FITW_WARPS = 8;
constexpr int FITW_U = 4;                       // loads in flight per lane

// Rare path of warp_lpr (num_lpr > 32, or more than 128 points tie below the bound): streaming selector with a
// bitonic sort of the candidate buffer. Kept out of line so that its ~2000 instructions stay out of the hot code.
__device__ __noinline__ double warp_lpr_fallback(const float4* __restrict__ P, int n, int nit, bool any_removed, const unsigned* __restrict__ alive_w,
                                                 float margin_f, int num_lpr, float* sel_buf) {
  const int lane = lane_id();
  double lpr = 0.0;
  LprSelector sel;
  sel.init(sel_buf, num_lpr);
  for (int it = 0; it < nit; ++it) {
    const int j = it * 32 + lane;
    bool valid = j < n;
    const float z = P[j < n ? j : n - 1].z;
    if (any_removed) valid = valid && ((alive_w[it] >> lane) & 1u);
    if (z < margin_f) valid = false;
    sel.push(valid, z);
  }
  sel.prune();
  if (lane == 0) {
    double sum = 0.0;
    for (int i = 0; i < sel.m; ++i) sum += (double) sel_buf[i];
    lpr = sel.m != 0 ? sum / sel.m : 0.0;
  }
  __syncwarp();
  return __shfl_sync(0xffffffffu, lpr, 0);
}

// LPR height for one warp-owned patch (extract_initial_seeds, S:84-103): mean of the (<= num_lpr) lowest z among
// the points that are alive and not below margin_f (float_ru of the zone-0 adaptive margin, -inf in the other zones).
// Two-level selection: the num_lpr-th smallest of the 32 per-lane minima is an upper bound T of the num_lpr-th
// smallest point, so only the few points with z <= T are gathered (ballot append into the warp's 128-slot buffer)
// and the exact k-th key is bisected among them. Falls back to the streaming selector when num_lpr > 32 or when
// more than 128 points tie below the bound.
__device__ double warp_lpr(const float4* __restrict__ P, int n, int nit, bool any_removed, const unsigned* __restrict__ alive_w, float margin_f,
                           int num_lpr, float* sel_buf) {
  const int lane = lane_id();
  const unsigned lt = lanemask_lt();
  unsigned* cbuf = reinterpret_cast<unsigned*>(sel_buf);
  bool fallback = num_lpr > 32;
  double lpr = 0.0;
  if (!fallback) {
    // (both scans: LPR_U loads in flight per lane. For class L1 the patch streams from L2 and these two loops were the kernel's top
    // long-scoreboard sites in a profile with one load per iteration; eight or four in flight cost more in code size than they hid —
    // the warp kernels stall on instruction fetch)
    constexpr int LPR_U = 2;
    unsigned kminL = 0xffffffffu;
    int nv = 0;
    for (int it0 = 0; it0 < nit; it0 += LPR_U) {
      float zb[LPR_U];
#pragma unroll
      for (int u = 0; u < LPR_U; ++u) { const int j = (it0 + u) * 32 + lane; zb[u] = P[j < n ? j : n - 1].z; }
#pragma unroll
      for (int u = 0; u < LPR_U; ++u) {
        const int it = it0 + u, j = it * 32 + lane;
        bool valid = j < n;
        const float z = zb[u];
        if (any_removed && it < nit) valid = valid && ((alive_w[it] >> lane) & 1u);
        if (z < margin_f) valid = false;
        if (valid) { kminL = min(kminL, order_key(z)); ++nv; }
      }
    }
    const int nvalid = __reduce_add_sync(0xffffffffu, nv);
    const int target = nvalid < num_lpr ? nvalid : num_lpr;
    if (target == 0) return 0.0;
    const int have = __reduce_add_sync(0xffffffffu, kminL != 0xffffffffu ? 1 : 0);
    unsigned T = 0xffffffffu;   // fewer lanes with candidates than target: keep everything
    if (have >= target) {
      const unsigned gmn = __reduce_min_sync(0xffffffffu, kminL);
      const unsigned gmx = __reduce_max_sync(0xffffffffu, kminL != 0xffffffffu ? kminL : 0u);
      T = kth_key(gmn, gmx, target, [&](unsigned cand) { return __reduce_add_sync(0xffffffffu, kminL < cand ? 1 : 0); });
    }
    int cc = 0;
    for (int it0 = 0; it0 < nit; it0 += LPR_U) {
      float zb[LPR_U];
#pragma unroll
      for (int u = 0; u < LPR_U; ++u) { const int j = (it0 + u) * 32 + lane; zb[u] = P[j < n ? j : n - 1].z; }
#pragma unroll
      for (int u = 0; u < LPR_U; ++u) {
        const int it = it0 + u, j = it * 32 + lane;
        bool valid = j < n;
        const float z = zb[u];
        if (any_removed && it < nit) valid = valid && ((alive_w[it] >> lane) & 1u);
        if (z < margin_f) valid = false;
        const unsigned key = order_key(z);
        const bool c = valid && key <= T;
        const unsigned bal = __ballot_sync(0xffffffffu, c);
        if (c) { const int pos = cc + __popc(bal & lt); if (pos < 128) cbuf[pos] = key; }
        cc += __popc(bal);
      }
    }
    __syncwarp();
    if (cc <= 128) {
      unsigned ck[4];
      unsigned kmn = 0xffffffffu, kmx = 0u;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = lane + 32 * q;
        ck[q] = i < cc ? cbuf[i] : 0xffffffffu;
        if (i < cc) { kmn = min(kmn, ck[q]); kmx = max(kmx, ck[q]); }
      }
      kmn = __reduce_min_sync(0xffffffffu, kmn);
      kmx = __reduce_max_sync(0xffffffffu, kmx);
      const unsigned ans = kth_key(kmn, kmx, target, [&](unsigned cand) {
        int cnt = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) cnt += ck[q] < cand;
        return __reduce_add_sync(0xffffffffu, cnt);
      });
      double ps = 0.0;
      int c_lt = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) if (ck[q] < ans) { ps += (double) key_to_float(ck[q]); ++c_lt; }
      ps = warp_sum(ps);
      c_lt = __reduce_add_sync(0xffffffffu, c_lt);
      lpr = (ps + (double) (target - c_lt) * (double) key_to_float(ans)) / (double) target;
      __syncwarp();
    } else fallback = true;
  }
  if (fallback) lpr = warp_lpr_fallback(P, n, nit, any_removed, alive_w, margin_f, num_lpr, sel_buf);
  return lpr;
}

// PLS: the current plane and the running moment sums of a warp's patch live in shared memory (160 B per warp) instead of ~40
// registers per lane: the passes only need the plane as four floats (PlaneF), the doubles are read in the rare exact distance
// test and by the solve. That is what lets the kernel run at 3 CTAs per SM (85 registers) without spilling.
template <bool STAGE, int CLS_HI, int CLS_LO, int U, int MINB, bool FUSE = false, bool PLS = false>
__global__ void __launch_bounds__(FITW_WARPS * 32, MINB) k_fit_warp(const float4* __restrict__ sorted, FrameTable ft, const StreamState* __restrict__ states,
                                                                             const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps, int nbp, const int* __restrict__ bin_off, WorkQueues wq,
                                                                             int* __restrict__ part, BinFit* __restrict__ fits) {
  constexpr int CAP = STAGE ? CLS_M_MAX : (CLS_HI == 2 ? CLS_L1_MAX : WARP_CAP);
  __shared__ unsigned s_alive[FITW_WARPS][CAP / 32];
  __shared__ unsigned s_member[FITW_WARPS][CAP / 32];
  __shared__ float s_sel[FITW_WARPS][128];
  __shared__ Plane s_pl[PLS ? FITW_WARPS : 1];
  __shared__ Moments s_tot[PLS ? FITW_WARPS : 1];
  static_assert(!(PLS && FUSE), "the fused seed round keeps two planes in registers");
  PW_DYN_SHARED(float4, s_stage);              // STAGE: [FITW_WARPS][CLS_M_MAX]
  const int warp = threadIdx.x >> 5, lane = lane_id();
  const unsigned lt = lanemask_lt();
  unsigned* alive_w = s_alive[warp];
  unsigned* member_w = s_member[warp];
  float* sel_buf = s_sel[warp];
  int cls = CLS_HI;          // queues being drained, longest patches first
  const int cls_last = CLS_LO;
  int cnt = wq.count[cls];
  const int4 no_item = make_int4(-1, 0, 0, 0);
  int4 cur = no_item;
  // synchronous claim: at the start and when a class runs dry. Inside the loop the warp claims one patch AHEAD (atomic at
  // the top of a patch, descriptor load after the first pass, L2 prefetch of its points before the R-GPF rounds), so
  // the queue round trips and most of the DRAM latency of the next patch overlap the current one.
  auto claim_sync = [&]() {
    cur = no_item;
    while (cls >= cls_last) {
      int t = 0;
      if (lane == 0) t = atomicAdd(&wq.head[cls], 1);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t < cnt) { cur = wq.items[cls][t]; return; }
      --cls;
      if (cls >= cls_last) cnt = wq.count[cls];
    }
  };
  claim_sync();

  for (;;) {
    if (cur.x < 0) return;
    int next_raw = 0;
    if (lane == 0) next_raw = atomicAdd(&wq.head[cls], 1);
    int4 nxt = no_item;
    bool looked_ahead = false;
    const int f = cur.x >> 12, bin = cur.x & 0xfff, n = cur.y;
    const int set = ft.pset[f];                  // the frame's parameter set
    const Geometry& g = gs.g[set];
    const AlgoParams& ap = aps.a[set];
    const float thf = (float) ap.th_dist;
    const long long start = work_item_start(cur);
    const float4* G = sorted + start;           // the patch in global memory
    int* out = part + start;
    const int nit = (n + 31) >> 5;
    const float4* P = G;                        // where the passes read the points from
    if (STAGE) {
      float4* mine = s_stage + warp * CLS_M_MAX;
      for (int it = 0; it < nit; it += FITW_U) {   // global loads: always FITW_U in flight
        float4 q[FITW_U];
#pragma unroll
        for (int u = 0; u < FITW_U; ++u) { const int j = (it + u) * 32 + lane; q[u] = G[j < n ? j : n - 1]; }
#pragma unroll
        for (int u = 0; u < FITW_U; ++u) { const int j = (it + u) * 32 + lane; if (j < n) mine[j] = q[u]; }
      }
      __syncwarp();
      P = mine;
    }
    const int zone = (bin >= g.bin_base[3]) ? 3 : (bin >= g.bin_base[2]) ? 2 : (bin >= g.bin_base[1]) ? 1 : 0;
    const bool zone0 = (zone == 0);
    // S:90; (double) z < margin  <=>  z < margin_f (float_ru), folded with the zone-0 condition
    const float margin_f = zone0 ? float_ru(ap.adaptive_seed_selection_margin * states[ft.stream[f]].sensor_height) : -INFINITY;
    const float4 first = P[0];
    double c[3] = {(double) first.x, (double) first.y, 0.0};   // reference point of all moment sums of this patch

    bool have_plane = false, any_removed = false;
    Plane pl_reg;
    Plane& pl = PLS ? s_pl[warp] : pl_reg;
    // PLS: every lane computes the same plane / sums; lane 0 stores them, a __syncwarp() publishes them
    auto set_plane = [&](const Plane& t) { if (!PLS) pl_reg = t; else { __syncwarp(); if (lane == 0) s_pl[warp] = t; __syncwarp(); } };
    {
      Plane z;
      z.d = 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) { z.mean[q] = 0.0; z.normal[q] = 0.0; z.sv[q] = 0.0; }
      set_plane(z);
    }

    // ---- seed rounds: R-VPF iterations (zone 0 only; for other zones the R-VPF fit is dead code, see k_fit_stream)
    //      followed by the R-GPF seed fit (S:484-514). Each is a selection pass + a full accumulation pass. ----
    Moments tot_reg;   // running sums of the current member set (valid after the last seed round)
    Moments& tot = PLS ? s_tot[warp] : tot_reg;
    auto set_tot = [&](const Moments& t) { if (!PLS) tot_reg = t; else { __syncwarp(); if (lane == 0) s_tot[warp] = t; __syncwarp(); } };
    int rvpf_left = (ap.enable_RVPF && zone0) ? ap.num_iter : 0;
    // FUSE: an R-VPF round that removes nothing is followed by the R-GPF seed fit over the SAME alive set with the
    // same margin, hence the same LPR height (S:84-103 depend on nothing else); its seed set {z < lpr + th_seeds} is a
    // subset of the R-VPF seed set {z < lpr + th_seeds_v} when th_seeds <= th_seeds_v. Such a round therefore
    // accumulates both sets in one pass (same summation order as two passes: bit-identical moments), solves the two
    // planes side by side in the two halves of the warp, and skips the second selection + pass when the R-VPF plane
    // turns out upright (the common case).
    const bool fuse_ok = FUSE && (ap.th_seeds <= ap.th_seeds_v);
    for (;;) {
      const bool rvpf_round = rvpf_left > 0;
      const bool fused = fuse_ok && rvpf_round;
      // LPR: mean of the num_lpr lowest z among the alive points not below the zone-0 margin (S:88-103)
      const double lpr = warp_lpr(P, n, nit, any_removed, alive_w, margin_f, ap.num_lpr, sel_buf);
      const float zthr = float_ru(lpr + (rvpf_round ? ap.th_seeds_v : ap.th_seeds));
      const float zin = float_ru(lpr + ap.th_seeds);   // inner (R-GPF seed) threshold of a fused round
      c[2] = lpr;
      if (!looked_ahead) {   // the claim issued at the top has returned by now: fetch the next patch's descriptor
        const int t_next = __shfl_sync(0xffffffffu, next_raw, 0);
        if (t_next < cnt) nxt = wq.items[cls][t_next];
        looked_ahead = true;
      }
      // full accumulation over {alive, z < lpr + th}; the ballots become the member set
      Moments m, mi;   // mi: the inner set of a fused round
      m.n = 0; mi.n = 0;
#pragma unroll
      for (int q = 0; q < 3; ++q) { m.s1[q] = 0.0; mi.s1[q] = 0.0; }
#pragma unroll
      for (int q = 0; q < 6; ++q) { m.s2[q] = 0.0; mi.s2[q] = 0.0; }
      for (int it = 0; it < nit; it += U) {
        float4 q[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int j = (it + u) * 32 + lane; q[u] = P[j < n ? j : n - 1]; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int j = (it + u) * 32 + lane;
          const float4 p = q[u];
          bool in = (j < n) && (p.z < zthr);                                              // S:108 / S:145
          if (any_removed && it + u < nit) in = in && ((alive_w[it + u] >> lane) & 1u);
          const unsigned bal = __ballot_sync(0xffffffffu, in);
          unsigned bal_in = bal;   // what becomes the member set: the inner set in a fused round
          bool inner = in;
          if (FUSE && fused) { inner = in && (p.z < zin); bal_in = __ballot_sync(0xffffffffu, inner); }
          if (lane == 0 && it + u < nit) member_w[it + u] = bal_in;
          if (bal) {
            const double w = in ? 1.0 : 0.0;   // unselected lanes add exact zeros
            const double dx = ((double) p.x - c[0]) * w, dy = ((double) p.y - c[1]) * w, dz = ((double) p.z - c[2]) * w;
            m.s1[0] += dx; m.s1[1] += dy; m.s1[2] += dz;
            m.s2[0] += dx * dx; m.s2[1] += dx * dy; m.s2[2] += dx * dz;
            m.s2[3] += dy * dy; m.s2[4] += dy * dz; m.s2[5] += dz * dz;
            m.n += in ? 1 : 0;
            if (FUSE && fused && bal_in) {
              const double wi = inner ? 1.0 : 0.0;
              const double ex = dx * wi, ey = dy * wi, ez = dz * wi;
              mi.s1[0] += ex; mi.s1[1] += ey; mi.s1[2] += ez;
              mi.s2[0] += ex * ex; mi.s2[1] += ex * ey; mi.s2[2] += ex * ez;
              mi.s2[3] += ey * ey; mi.s2[4] += ey * ez; mi.s2[5] += ez * ez;
              mi.n += inner ? 1 : 0;
            }
          }
        }
      }
      group_sum_moments<32>(m, lane);
      m.n = warp_sum_i(m.n);
      if (FUSE && fused) {
        group_sum_moments<32>(mi, lane);
        mi.n = warp_sum_i(mi.n);
        // lanes 0..15 solve the R-VPF plane (all seeds), lanes 16..31 the R-GPF seed plane (inner seeds)
        const bool hi = lane >= 16;
        Moments ms;
        ms.n = hi ? mi.n : m.n;
#pragma unroll
        for (int q = 0; q < 3; ++q) ms.s1[q] = hi ? mi.s1[q] : m.s1[q];
#pragma unroll
        for (int q = 0; q < 6; ++q) ms.s2[q] = hi ? mi.s2[q] : m.s2[q];
        Plane mine = pl;
        if (ms.n > 0) plane_from_moments(ms, c, mine);
        auto bcast = [&](int src) {
          Plane t;
#pragma unroll
          for (int q = 0; q < 3; ++q) { t.mean[q] = __shfl_sync(0xffffffffu, mine.mean[q], src); t.normal[q] = __shfl_sync(0xffffffffu, mine.normal[q], src); t.sv[q] = __shfl_sync(0xffffffffu, mine.sv[q], src); }
          t.d = __shfl_sync(0xffffffffu, mine.d, src);
          return t;
        };
        if (m.n > 0) { pl = bcast(0); have_plane = true; }     // the R-VPF fit (S:486); S:49 keeps the previous plane otherwise
        if (!(have_plane && pl.normal[2] < ap.uprightness_thr)) {   // S:506 break: nothing removed, the seed fit follows
          if (mi.n > 0) { pl = bcast(16); have_plane = true; }  // S:513-514 on the same alive set
          set_tot(mi);
          break;
        }
      } else {
        if (m.n > 0) { Plane t; plane_from_moments(m, c, t); set_plane(t); have_plane = true; }   // S:49: an empty set keeps the previous plane
        set_tot(m);
        if (!rvpf_round) break;
      }
      if (have_plane && pl.normal[2] < ap.uprightness_thr) {   // S:489: remove the vertical structure, iterate
        for (int it = 0; it < nit; ++it) {
          const int j = it * 32 + lane;
          bool keep = j < n;
          const float4 p = P[j < n ? j : n - 1];
          if (any_removed) keep = keep && ((alive_w[it] >> lane) & 1u);
          const bool was_alive = keep;
          keep = keep && !(fabs(point_plane_distance(pl, p.x, p.y, p.z)) < ap.th_dist_v);   // S:499
          if (wq.labels && was_alive && !keep) wq.labels[start + j] = (unsigned char) (ap.num_iter - rvpf_left + 1);
          const unsigned bal = __ballot_sync(0xffffffffu, keep);
          if (lane == 0) alive_w[it] = bal;
        }
        __syncwarp();
        any_removed = true;
        --rvpf_left;
      } else rvpf_left = 0;   // S:506 break
    }
    __syncwarp();

    if (nxt.x >= 0) prefetch_patch_l2(sorted + work_item_start(nxt), nxt.y, lane, 32);
    // ---- R-GPF iterations (S:516-543): num_iter distance passes; incremental moments; stop at the fixpoint ----
    for (int round = 0; round < ap.num_iter && have_plane; ++round) {
      PlaneF pf;
      pf.n0 = (float) pl.normal[0]; pf.n1 = (float) pl.normal[1]; pf.n2 = (float) pl.normal[2]; pf.d = (float) pl.d;
      Moments dm;
      dm.n = 0;
#pragma unroll
      for (int q = 0; q < 3; ++q) dm.s1[q] = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) dm.s2[q] = 0.0;
      unsigned changed_any = 0;
      for (int it = 0; it < nit; it += U) {
        float4 q[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int j = (it + u) * 32 + lane; q[u] = P[j < n ? j : n - 1]; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (it + u >= nit) break;
          const int j = (it + u) * 32 + lane;
          const float4 p = q[u];
          int fl = dist_filter(pf, thf, p.x, p.y, p.z);
          if (fl < 0) fl = (point_plane_distance(pl, p.x, p.y, p.z) < ap.th_dist) ? 1 : 0;   // S:525 / S:529, exact
          bool in = (j < n) && (fl != 0);
          if (any_removed) in = in && ((alive_w[it + u] >> lane) & 1u);
          const unsigned bal = __ballot_sync(0xffffffffu, in);
          const unsigned prev = member_w[it + u];
          const unsigned chg = bal ^ prev;
          if (chg) {   // warp-uniform: only iterations with a membership change touch the double-precision sums
            changed_any |= chg;
            const bool mine = (chg >> lane) & 1u;
            const double w = mine ? (in ? 1.0 : -1.0) : 0.0;
            const double dx = (double) p.x - c[0], dy = (double) p.y - c[1], dz = (double) p.z - c[2];
            const double wx = dx * w, wy = dy * w, wz = dz * w;
            dm.s1[0] += wx; dm.s1[1] += wy; dm.s1[2] += wz;
            dm.s2[0] += wx * dx; dm.s2[1] += wx * dy; dm.s2[2] += wx * dz;
            dm.s2[3] += wy * dy; dm.s2[4] += wy * dz; dm.s2[5] += wz * dz;
            dm.n += mine ? (in ? 1 : -1) : 0;
            __syncwarp();
            if (lane == 0) member_w[it + u] = bal;
          }
        }
      }
      if (changed_any == 0) break;   // fixpoint: every later iteration would reproduce this set and this plane
      {
        group_sum_moments<32>(dm, lane);
        Moments t = tot;
#pragma unroll
        for (int q = 0; q < 3; ++q) t.s1[q] += dm.s1[q];
#pragma unroll
        for (int q = 0; q < 6; ++q) t.s2[q] += dm.s2[q];
        t.n += warp_sum_i(dm.n);
        set_tot(t);
        if (t.n > 0) { Plane np; plane_from_moments(t, c, np); set_plane(np); }   // S:49 otherwise
      }
      __syncwarp();
    }
    const int n_ground = have_plane ? tot.n : 0;
    __syncwarp();
    // stable partition: ground indices ascending, then non-ground indices ascending
    {
      int g_run = 0, ng_run = 0;
      for (int it0 = 0; it0 < nit; it0 += U) {   // U index loads in flight per lane
        int idxb[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int j = (it0 + u) * 32 + lane; idxb[u] = __float_as_int(P[j < n ? j : n - 1].w); }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int it = it0 + u, j = it * 32 + lane;
          if (it >= nit) break;
          const bool v = j < n;
          const unsigned bg = have_plane ? member_w[it] : 0u;
          const unsigned bv = __ballot_sync(0xffffffffu, v);
          const unsigned bn = bv & ~bg;
          if (v) {
            const int idx = idxb[u];
            if ((bg >> lane) & 1u) out[g_run + __popc(bg & lt)] = idx;
            else out[n_ground + ng_run + __popc(bn & lt)] = idx;
            if (wq.labels) { const bool isg = (bg >> lane) & 1u; if (isg || !any_removed || ((alive_w[it] >> lane) & 1u)) wq.labels[start + j] = isg ? PW_LABEL_GROUND : PW_LABEL_REJECT; }
          }
          g_run += __popc(bg);
          ng_run += __popc(bn);
        }
      }
    }
    if (lane == 0) {
      BinFit& r = fits[(size_t) f * gs.nbs + bin];
      r.n = n; r.n_ground = n_ground; r.fitted = 1;
      r.verdict = have_plane ? 0 : PW_FIT_NO_PLANE;
#pragma unroll
      for (int q = 0; q < 3; ++q) { r.mean[q] = pl.mean[q]; r.normal[q] = pl.normal[q]; r.sv[q] = pl.sv[q]; }
      r.d = pl.d;
    }
    __syncwarp();
    if (nxt.x >= 0) cur = nxt;
    else {   // this class is drained (the look-ahead claim ran past its end): continue with the next one
      --cls;
      if (cls >= cls_last) cnt = wq.count[cls];
      claim_sync();
    }
  }
}

}  // namespace pwpp

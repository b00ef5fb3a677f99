// pwpp_fit_ref32.cuh — the plane fits in the reference's own arithmetic (pwpp_set_arithmetic(ctx, PWPP_ARITH_REFERENCE)).
//
// Reference: cpp/patchworkpp/src/patchworkpp.cpp ("S:") 467-549 (extract_piecewiseground), 77-149 (extract_initial_seeds),
// 47-75 (estimate_plane), 551-554 (calc_point_to_plane_d), and the per-bin sort of S:199.
//
// The other fit kernels (pwpp_fit.cuh) evaluate the fits in double with order-free sums. The reference sums in fp32, point
// after point, in the z-sorted order of the bin: its rounding depends on that order. This kernel runs S:467-549 literally:
//   - the patch is sorted by (z, tie key) on chip, -0 and +0 as one z, as the reference's comparator sees them. The tie key is
//     the position in the bin, which holds its points in ascending index order: equal z keep ascending point index, the order
//     std::stable_sort gives (libpwref_stable.so). Under PWPP_ORDER_REFERENCE_EXACT (exact_ties) a patch with equal z takes as tie
//     key each point's position after libstdc++'s introsort loop (ox_warp_loop of pwpp_order_exact.cuh, run by warp 0), so equal
//     z are in std::sort's order (libpwref.so): std::sort is that loop followed by a stable insertion sort;
//   - every estimate_plane compacts its point set in that order and sums it on single threads: 3 sequential fp32 chains
//     for the mean, then 6 for the covariance, then the fp32 Jacobi SVD of pwpp_math.cuh on one thread;
//   - every per-point step (distances, removal masks, seed predicates, prefix counts) runs on all threads of the CTA;
//   - the LPR height is the double sum of at most num_lpr floats in sorted order, on one thread.
// Every floating-point operation is separately rounded (fadd / fmul / ... of pwpp_math.cuh): no contraction.
//
// One CTA per patch, persistent over one class queue (the queues k_bin_scan / k_front_cluster fill). A patch of at most CAP
// points lives in shared memory; a larger one (dense sensors: bins of 20k-40k points) in a global scratch at its own offset
// into the bin-sorted array, so no two patches of a call share scratch. The kernel writes `part`, `labels` and the BinFit
// record exactly as the other fit kernels define them, so k_order, k_order_exact, k_gle and k_emit run unchanged.
// The two defined deviations stay: a patch whose every point set was empty gets PW_FIT_NO_PLANE (k_gle then carries the last
// plane), and a missing plane selects no point.
#pragma once
#include <cuda_runtime.h>

#include "pwpp_fit.cuh"
#include "pwpp_order_exact.cuh"

namespace pwpp {

// Global storage of the patches above a kernel's CAP points, indexed by the patch's offset into the bin-sorted array.
struct Ref32Scratch {
  unsigned long long* keys;   // [2 * points]: sort keys, the power-of-two padding of a patch of n points fits in 2n
  float4* pts;                // [points]: the patch in sorted order, w = position in the bin
  float* sel;                 // [3 * points]: x, y, z planes of the point set of the current fit
  unsigned char* flags;       // [2 * points]: per sorted point what became of it, then per position its ground flag
};
// the sort key of a z value: -0 and +0 are one key, as for the reference's comparator
__device__ __forceinline__ unsigned long long ref32_zkey(float z) { if (z == 0.f) z = 0.f; return (unsigned long long) order_key(z) << 32; }
// shared memory of a kernel with capacity CAP (a power of two)
__host__ __device__ constexpr size_t ref32_smem_bytes(int cap) { return (size_t) cap * (8 + 16 + 12 + 2); }
constexpr int R32_SMALL_CAP = 512, R32_BIG_CAP = 2048;

// fp32 point-plane distance plus d in double, S:551-554
__device__ __forceinline__ double ref32_dist(const float4& p, float n0, float n1, float n2, double d) {
  return dadd((double) fadd(fadd(fmul(n0, p.x), fmul(n1, p.y)), fmul(n2, p.z)), d);
}

// S:62-74 on one thread from the 6 covariance entries and the mean: the plane's normal (z >= 0), singular values and d.
// Not inlined: every estimate_plane of the kernel calls it, and one copy of the Jacobi iteration keeps the kernel small.
__device__ __noinline__ void ref32_solve(const float* cv, const float* mean, float* nrm, float* svo, double* d) {
  const float cov[9] = {cv[0], cv[1], cv[2], cv[1], cv[3], cv[4], cv[2], cv[4], cv[5]};
  float sv[3], U[9];
  jacobi_svd3f(cov, sv, U);
  float nr[3] = {U[6], U[7], U[8]};
  if (nr[2] < 0.f) for (int q = 0; q < 3; ++q) nr[q] = -nr[q];
  const float x0 = fmul(nr[0], mean[0]), x1 = fmul(nr[1], mean[1]), x2 = fmul(nr[2], mean[2]);
  *d = -(double) fadd(x0, fadd(x1, x2));
  for (int q = 0; q < 3; ++q) { nrm[q] = nr[q]; svo[q] = sv[q]; }
}

template <int CLS, int NT, int CAP>
__global__ void __launch_bounds__(NT, 1) k_fit_ref32(const float4* __restrict__ sorted, FrameTable ft, const StreamState* __restrict__ states,
                                                  const __grid_constant__ GeometrySets gs, const __grid_constant__ AlgoParamSets aps, const int* __restrict__ bin_off,
                                                  WorkQueues wq, int* __restrict__ part, BinFit* __restrict__ fits, Ref32Scratch scr,
                                                  int exact_ties) {
  constexpr int NW = NT / 32;
  static_assert((CAP & (CAP - 1)) == 0, "CAP is a power of two");
  PW_DYN_SHARED(unsigned long long, s_dyn);
  __shared__ int4 s_item;
  __shared__ int s_wcnt[2][NW];         // per-warp counts of a block scan, double-buffered by chunk parity
  __shared__ float s_mean[3];
  __shared__ float s_cov[6];
  __shared__ float s_nrm[3], s_sv[3];
  __shared__ double s_d, s_lpr;
  __shared__ int s_have;
  __shared__ int s_tie;
  __shared__ int s_ox_stk[OX_STACK * 3];   // the stack of the introsort loop (exact_ties)
  __shared__ float s_lz[MAX_LPR];       // z of the LPR points in sorted order
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const unsigned lt = lanemask_lt();
  const int count = wq.count[CLS];

  for (;;) {
    if (tid == 0) {
      const int t = atomicAdd(&wq.head[CLS], 1);
      s_item = t < count ? wq.items[CLS][t] : make_int4(-1, 0, 0, 0);
    }
    __syncthreads();
    const int4 cur = s_item;
    if (cur.x < 0) return;
    const int f = cur.x >> 12, bin = cur.x & 0xfff, n = cur.y;
    const AlgoParams& ap = aps.a[ft.pset[f]];
    const Geometry& g = gs.g[ft.pset[f]];
    const long long start = work_item_start(cur);
    const float4* P = sorted + start;
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    // patch storage: shared memory up to CAP points, else the patch's own region of the global scratch
    unsigned long long* keys;
    float4* pts;
    float *cx, *cy, *cz;
    unsigned char *lab, *gpos;
    if (n <= CAP) {
      keys = s_dyn;
      pts = reinterpret_cast<float4*>(keys + CAP);
      cx = reinterpret_cast<float*>(pts + CAP); cy = cx + CAP; cz = cy + CAP;
      lab = reinterpret_cast<unsigned char*>(cz + CAP); gpos = lab + CAP;
    } else {
      keys = scr.keys + 2 * start;
      pts = scr.pts + start;
      cx = scr.sel + 3 * start; cy = cx + n; cz = cy + n;
      lab = scr.flags + 2 * start; gpos = lab + n;
    }

    // ---- S:199: sort by (z, tie key) ----
    auto sort_keys = [&]() {   // bitonic, ascending, over keys[0, np2)
      for (int k = 2; k <= np2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int i = tid; i < np2; i += NT) {
            const int l = i ^ j;
            if (l > i) {
              const unsigned long long a = keys[i], b = keys[l];
              if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[l] = a; }
            }
          }
          __syncthreads();
        }
    };
    for (int i = tid; i < np2; i += NT) keys[i] = i < n ? (ref32_zkey(P[i].z) | (unsigned) i) : ~0ull;
    if (tid == 0) s_tie = 0;
    __syncthreads();
    sort_keys();
    // position in the bin of the point with tie key t: t itself, or inv[t] after the introsort loop
    const int* inv = nullptr;
    if (exact_ties) {
      for (int r = tid; r + 1 < n; r += NT)
        if ((keys[r] >> 32) == (keys[r + 1] >> 32)) s_tie = 1;
      __syncthreads();
      if (s_tie) {
        // the loop over the bin's z in bin order (what the reference sorts); workspace: the pts region (4n words), then the
        // loop's output sequence in the cx region
        float* zk = reinterpret_cast<float*>(pts);
        int* sq = reinterpret_cast<int*>(pts) + n;
        int* ix = reinterpret_cast<int*>(pts) + 2 * n;
        for (int i = tid; i < n; i += NT) { zk[i] = P[i].z; sq[i] = i; }
        __syncthreads();
        if (w == 0 && n > OX_THRESHOLD) ox_warp_loop(zk, sq, ix, n, s_ox_stk, 0, n, 2 * (31 - __clz(n)), nullptr);
        __syncthreads();
        int* sqo = reinterpret_cast<int*>(cx);
        for (int q = tid; q < np2; q += NT) {
          if (q < n) sqo[q] = sq[q];
          keys[q] = q < n ? (ref32_zkey(zk[q]) | (unsigned) q) : ~0ull;
        }
        __syncthreads();
        sort_keys();
        inv = sqo;
      }
    }
    for (int r = tid; r < n; r += NT) {
      const int t = (int) (unsigned) keys[r];
      const int j = inv ? inv[t] : t;
      const float4 p = P[j];
      pts[r] = make_float4(p.x, p.y, p.z, __int_as_float(j));
      lab[r] = 0;   // 0: alive; 1..num_iter: removed by that R-VPF iteration; PW_LABEL_GROUND: ground
    }
    if (tid == 0) { s_have = 0; s_d = 0.0; for (int q = 0; q < 3; ++q) { s_nrm[q] = 0.f; s_mean[q] = 0.f; s_sv[q] = 0.f; } }
    __syncthreads();

    // Block-wide compaction in sorted order: pred(r) is evaluated once per point; on(r, pos) runs for every selected point with
    // its rank among them. Returns the number selected (uniform).
    auto compact = [&](auto pred, auto on) -> int {
      int base = 0, par = 0;
      for (int c0 = 0; c0 < n; c0 += NT, par ^= 1) {
        const int r = c0 + tid;
        const bool in = r < n && pred(r);
        const unsigned b = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_wcnt[par][w] = __popc(b);
        __syncthreads();
        int off = 0, tot = 0;
#pragma unroll
        for (int q = 0; q < NW; ++q) { const int v = s_wcnt[par][q]; off += q < w ? v : 0; tot += v; }
        if (in) on(r, base + off + __popc(b & lt));
        base += tot;
      }
      __syncthreads();
      return base;
    };
    // estimate_plane S:47-75 on the m points in cx / cy / cz; an empty set keeps the plane (S:49)
    auto fit_selected = [&](int m) {
      if (m == 0) return;
      if (tid < 3) {
        const float* c = tid == 0 ? cx : tid == 1 ? cy : cz;
        float s = 0.f;
        for (int i = 0; i < m; ++i) s = fadd(s, c[i]);
        s_mean[tid] = fdiv(s, (float) m);
      }
      __syncthreads();
      if (tid < 6) {   // xx xy xz yy yz zz
        const int a = tid < 3 ? 0 : tid < 5 ? 1 : 2, b = tid < 3 ? tid : tid < 5 ? tid - 2 : 2;
        const float* ca = a == 0 ? cx : a == 1 ? cy : cz;
        const float* cb = b == 0 ? cx : b == 1 ? cy : cz;
        const float ma = s_mean[a], mb = s_mean[b];
        float s = 0.f;
        for (int i = 0; i < m; ++i) s = fadd(s, fmul(fsub(ca[i], ma), fsub(cb[i], mb)));
        s_cov[tid] = fdiv(s, (float) (double) (m - 1));
      }
      __syncthreads();
      if (tid == 0) { ref32_solve(s_cov, s_mean, s_nrm, s_sv, &s_d); s_have = 1; }
      __syncthreads();
    };
    auto take = [&](int r, int pos) { const float4 p = pts[r]; cx[pos] = p.x; cy[pos] = p.y; cz[pos] = p.z; };
    const int zone = (bin >= g.bin_base[3]) ? 3 : (bin >= g.bin_base[2]) ? 2 : (bin >= g.bin_base[1]) ? 1 : 0;
    const double margin = dmul(ap.adaptive_seed_selection_margin, states[ft.stream[f]].sensor_height);
    // extract_initial_seeds S:77-149 over the alive points: the LPR height
    auto lpr_height = [&]() -> double {
      int init_idx = 0;
      if (zone == 0) init_idx = compact([&](int r) { return lab[r] == 0 && (double) pts[r].z < margin; }, [](int, int) {});
      const int lo = init_idx, hi = init_idx + ap.num_lpr;
      const int alive = compact([&](int r) { return lab[r] == 0; }, [&](int r, int pos) { if (pos >= lo && pos < hi) s_lz[pos - lo] = pts[r].z; });
      if (tid == 0) {
        const int cnt = min(ap.num_lpr, max(alive - init_idx, 0));
        double sum = 0.0;
        for (int k = 0; k < cnt; ++k) sum = dadd(sum, (double) s_lz[k]);
        s_lpr = cnt != 0 ? ddiv(sum, (double) cnt) : 0.0;
      }
      __syncthreads();
      return s_lpr;
    };
    auto seeds = [&](double lpr, double th) {
      const double t = dadd(lpr, th);
      return compact([&](int r) { return lab[r] == 0 && (double) pts[r].z < t; }, take);
    };
    auto dist = [&](int r) { return ref32_dist(pts[r], s_nrm[0], s_nrm[1], s_nrm[2], s_d); };

    // ---- S:481-509 R-VPF ----
    if (ap.enable_RVPF && zone == 0) {
      for (int it = 0; it < ap.num_iter; ++it) {
        fit_selected(seeds(lpr_height(), ap.th_seeds_v));
        if (!(s_have && (double) s_nrm[2] < ap.uprightness_thr)) break;
        for (int r = tid; r < n; r += NT)
          if (lab[r] == 0 && fabs(dist(r)) < ap.th_dist_v) lab[r] = (unsigned char) (it + 1);
        __syncthreads();
      }
    }
    // ---- S:511-513 the R-GPF seed plane. Outside zone 0 the R-VPF loop fits the th_seeds_v seeds once and breaks; that plane
    // is only seen when the th_seeds seed set is empty (same LPR height: the point set is the same), so it is fitted then ----
    {
      const double lpr = lpr_height();
      int m = seeds(lpr, ap.th_seeds);
      if (m == 0 && ap.enable_RVPF && zone != 0) m = seeds(lpr, ap.th_seeds_v);
      fit_selected(m);
    }
    // ---- S:515-547 R-GPF: num_iter - 1 refits, then the final split and its plane ----
    for (int it = 0; it < ap.num_iter; ++it) {
      const bool last = it == ap.num_iter - 1;
      const bool have = s_have != 0;
      const int m = compact([&](int r) { return lab[r] == 0 && have && dist(r) < ap.th_dist; },
                            [&](int r, int pos) { take(r, pos); if (last) lab[r] = PW_LABEL_GROUND; });
      fit_selected(m);
    }

    // ---- outputs: labels, part (ground ascending by index, then non-ground), the patch record ----
    for (int r = tid; r < n; r += NT) {
      const int j = __float_as_int(pts[r].w);
      const unsigned char l = lab[r];
      gpos[j] = l == PW_LABEL_GROUND;
      if (wq.labels) wq.labels[start + j] = l;   // PW_LABEL_REJECT is 0: an alive point that is not ground
    }
    __syncthreads();
    int* out = part + start;
    const int n_ground = compact([&](int j) { return gpos[j] != 0; }, [&](int j, int pos) { out[pos] = __float_as_int(P[j].w); });
    compact([&](int j) { return gpos[j] == 0; }, [&](int j, int pos) { out[n_ground + pos] = __float_as_int(P[j].w); });
    if (tid == 0) {
      BinFit& rec = fits[(size_t) f * gs.nbs + bin];
      rec.n = n; rec.n_ground = n_ground; rec.fitted = 1;
      rec.verdict = s_have ? 0 : PW_FIT_NO_PLANE;
      for (int q = 0; q < 3; ++q) { rec.mean[q] = s_mean[q]; rec.normal[q] = s_nrm[q]; rec.sv[q] = s_sv[q]; }
      rec.d = s_d;
    }
    __syncthreads();
  }
}

}  // namespace pwpp

// pwpp_order_exact.cuh — the unmodified reference's order of equal z (optional stage, pwpp_set_output_order(PWPP_ORDER_REFERENCE_EXACT)).
//
// k_order (pwpp_order.cuh) puts every fitted patch's parts in the reference's order (group, z) and breaks ties in z by ascending
// point index: the order of a STABLE per-bin sort. The reference sorts its bins with std::sort (S:199), and libstdc++'s std::sort
// leaves equal z in an order of its own. This stage runs after k_order on the same work queues and reproduces that order.
//
// libstdc++'s std::sort is an introsort loop followed by one insertion sort over the whole range. The insertion sort is stable, and
// the loop leaves segments that are ordered against each other, so for a comparator that is a strict weak order (no NaN z) the
// result is the STABLE sort by z of the sequence the loop leaves behind: among equal z, the element's position q after the loop
// decides. The loop itself, on a segment [l, h) of more than 16 elements at depth d (2 floor(log2 n) at the start):
//   d == 0 : heap sort of the segment (make_heap + sort_heap);
//   else   : the median of (l+1, l+(h-l)/2, h-1) is moved to l (its exact sequence of compares), p = a[l]; with L_k the k-th position
//            of [l+1, h) from the left with !(a < p) and R_k the k-th from the right with !(p < a), the Hoare partition swaps
//            a[L_k] and a[R_k] for every k with L_k < R_k (K of them) and cuts at min(L_{K+1}, R_K) (R_0 = h); both halves go on at
//            depth d - 1.
// The segments are disjoint, so they are processed in any order. Steps L and R are two prefix counts: a partition is a team-wide
// scan of the two stopper kinds, a scatter of their positions, a binary search for K and K parallel swaps.
//
// Per patch, one warp:
//   1. tie check: the parts k_order wrote, read back through the positions of their points; a patch in which no two neighbours
//      of one group have equal z (and no z is NaN) is left as it is;
//   2. the introsort loop over the bin's z in point order (what the reference sorts), segment by segment, depth first; each
//      partition from ballots of the two stopper kinds and their warp prefix counts; the heap branch runs in one lane;
//   3. the parts rewritten in the order (group, z, q) — one sort of 64-bit keys.
// A bin with a NaN z is not sorted by a strict weak order; there one thread runs the whole of std::sort, insertion sort included,
// and the parts are rewritten in the order (group, position in its output).
// Workspace: shared memory for classes S and M (up to 512 points); the larger classes use a global scratch of OX_X_WORDS words per
// point of the call, each patch the region at its start.
#pragma once
#include "pwpp_order.cuh"

namespace pwpp {

constexpr int OX_THRESHOLD = 16;    // libstdc++'s _S_threshold: shorter segments are left to the final insertion sort
constexpr int OX_STACK = 64;        // pending segments of one warp (depth-first: at most the depth limit, 2 floor(log2 n) < 48, plus one)
constexpr int OX_X_WORDS = 4;       // scratch of the classes above 512 points, 32-bit words per point of the call
constexpr int OX_NUM_STATS = 3;     // counters: patches simulated, heap fall-backs, NaN bins

// workspace of a patch of n points in 32-bit words: z, sequence, two stopper-position arrays (after the loop: the 64-bit sort
// keys); even, so that the key array stays 8-byte aligned
__host__ __device__ constexpr size_t ox_ws_words(long long n) { return (size_t) ((4 * n + 1) & ~1ll); }
constexpr int OX_WARP_THREADS = 128;
__host__ __device__ constexpr size_t ox_warp_smem_bytes() { return (size_t) (OX_WARP_THREADS / 32) * (ox_ws_words(CLS_M_MAX) + 3 * OX_STACK) * 4; }

// ---- the team of a patch: one warp ----
struct OxWarp {
  static constexpr int size = 32;
  __device__ __forceinline__ int rank() const { return threadIdx.x & 31; }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ bool any(bool p) const { return __any_sync(0xffffffffu, p) != 0; }
  // exclusive prefix sums of a and b over the team, and their totals
  __device__ __forceinline__ void scan2(int a, int b, int& ea, int& eb, int& ta, int& tb) const {
    int x = a, y = b;
    const int lane = rank();
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, x, d), v = __shfl_up_sync(0xffffffffu, y, d);
      if (lane >= d) { x += u; y += v; }
    }
    ta = __shfl_sync(0xffffffffu, x, 31);
    tb = __shfl_sync(0xffffffffu, y, 31);
    ea = x - a;
    eb = y - b;
  }
};
// ---- the literal algorithm, one thread (heap branch, NaN bins) ----
__device__ __forceinline__ void ox_swap(float* zk, int* sq, int i, int j) {
  const float z = zk[i]; zk[i] = zk[j]; zk[j] = z;
  const int s = sq[i]; sq[i] = sq[j]; sq[j] = s;
}
// median of the elements at a, b, c moved to r, by libstdc++'s sequence of compares
__device__ __forceinline__ void ox_median_to_first(float* zk, int* sq, int r, int a, int b, int c) {
  const float za = zk[a], zb = zk[b], zc = zk[c];
  int m;
  if (za < zb) m = zb < zc ? b : (za < zc ? c : a);
  else m = za < zc ? a : (zb < zc ? c : b);
  ox_swap(zk, sq, r, m);
}
// sift the value (z, s) down from hole in a heap of len elements at base, then up to top
__device__ __forceinline__ void ox_adjust_heap(float* zk, int* sq, int base, int hole, int len, float z, int s) {
  const int top = hole;
  int child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (zk[base + child] < zk[base + child - 1]) --child;
    zk[base + hole] = zk[base + child]; sq[base + hole] = sq[base + child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    zk[base + hole] = zk[base + child - 1]; sq[base + hole] = sq[base + child - 1];
    hole = child - 1;
  }
  int parent = (hole - 1) / 2;
  while (hole > top && zk[base + parent] < z) {
    zk[base + hole] = zk[base + parent]; sq[base + hole] = sq[base + parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  zk[base + hole] = z; sq[base + hole] = s;
}
__device__ __forceinline__ void ox_heap_sort(float* zk, int* sq, int l, int h) {
  const int len = h - l;
  for (int parent = (len - 2) / 2; len >= 2; --parent) {
    ox_adjust_heap(zk, sq, l, parent, len, zk[l + parent], sq[l + parent]);
    if (parent == 0) break;
  }
  for (int last = h - 1; last - l >= 1; --last) {   // pop: the root goes to last, the old last value sifts down from the root
    const float z = zk[last];
    const int s = sq[last];
    zk[last] = zk[l]; sq[last] = sq[l];
    ox_adjust_heap(zk, sq, l, 0, last - l, z, s);
  }
}
// the unguarded partition of [l + 1, h) around a[l], kept inside the segment (a NaN z can walk the reference's scans out of it)
__device__ __forceinline__ int ox_partition_serial(float* zk, int* sq, int l, int h) {
  ox_median_to_first(zk, sq, l, l + 1, l + (h - l) / 2, h - 1);
  const float p = zk[l];
  int first = l + 1, last = h;
  for (;;) {
    while (first < h - 1 && zk[first] < p) ++first;
    --last;
    while (last > l && p < zk[last]) --last;
    if (!(first < last)) return first;
    ox_swap(zk, sq, first, last);
    ++first;
  }
}
// the whole of std::sort over [0, n), insertion sort included; stk: OX_STACK * 3 words
__device__ __forceinline__ void ox_std_sort_serial(float* zk, int* sq, int n, int* stk, unsigned long long* stats) {
  if (n < 2) return;
  int top = 0;
  stk[0] = 0; stk[1] = n; stk[2] = 2 * (31 - __clz(n)); top = 1;
  while (top > 0) {
    --top;
    const int l = stk[3 * top], d = stk[3 * top + 2];
    int h = stk[3 * top + 1];
    if (h - l <= OX_THRESHOLD) continue;
    if (d == 0) {
      ox_heap_sort(zk, sq, l, h);
      if (stats) atomicAdd(stats + 1, 1ull);
      continue;
    }
    const int cut = ox_partition_serial(zk, sq, l, h);
    stk[3 * top] = cut; stk[3 * top + 1] = h; stk[3 * top + 2] = d - 1; ++top;
    stk[3 * top] = l; stk[3 * top + 1] = cut; stk[3 * top + 2] = d - 1; ++top;
  }
  auto linear_insert = [&](int i) {
    const float z = zk[i];
    const int s = sq[i];
    while (i > 0 && z < zk[i - 1]) { zk[i] = zk[i - 1]; sq[i] = sq[i - 1]; --i; }
    zk[i] = z; sq[i] = s;
  };
  const int head = n > OX_THRESHOLD ? OX_THRESHOLD : n;
  for (int i = 1; i < head; ++i) {
    if (zk[i] < zk[0]) {   // to the front, everything before it one place up
      const float z = zk[i];
      const int s = sq[i];
      for (int k = i; k > 0; --k) { zk[k] = zk[k - 1]; sq[k] = sq[k - 1]; }
      zk[0] = z; sq[0] = s;
    } else {
      linear_insert(i);
    }
  }
  for (int i = head; i < n; ++i) linear_insert(i);
}

// ---- the introsort loop by teams ----
// One partition step of [l, h) (h - l > OX_THRESHOLD, depth > 0) by the team; ixl / ixr: scratch of h - l words each. Returns the cut.
template <class Team>
__device__ __forceinline__ int ox_partition(const Team& tm, float* zk, int* sq, int* ixl, int* ixr, int l, int h) {
  if (tm.rank() == 0) ox_median_to_first(zk, sq, l, l + 1, l + (h - l) / 2, h - 1);
  tm.sync();
  const float p = zk[l];
  const int per = (h - l - 1 + Team::size - 1) / Team::size;
  const int b0 = min(h, l + 1 + tm.rank() * per), b1 = min(h, b0 + per);
  int cl = 0, cr = 0;
  for (int j = b0; j < b1; ++j) { const float v = zk[j]; cl += !(v < p); cr += !(p < v); }
  int el, er, tl, tr;
  tm.scan2(cl, cr, el, er, tl, tr);
  for (int j = b0; j < b1; ++j) {
    const float v = zk[j];
    if (!(v < p)) ixl[el++] = j;                  // L_(el+1), 0-based el
    if (!(p < v)) { ixr[tr - 1 - er] = j; ++er; }  // counted from the right
  }
  tm.sync();
  int lo = 0, hi = min(tl, tr);   // K = the number of k with L_k < R_k, a prefix of k
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ixl[mid] < ixr[mid]) lo = mid + 1;
    else hi = mid;
  }
  const int K = lo;
  const int cut = min(K < tl ? ixl[K] : h, K > 0 ? ixr[K - 1] : h);
  for (int k = tm.rank(); k < K; k += Team::size) ox_swap(zk, sq, ixl[k], ixr[k]);
  tm.sync();
  return cut;
}

// One warp runs the loop from segment [l, h) at depth d to its end, depth first; stk: the warp's OX_STACK * 3 words.
__device__ __forceinline__ void ox_warp_loop(float* zk, int* sq, int* ix, int n, int* stk, int l, int h, int d, unsigned long long* stats) {
  const OxWarp wp;
  const int lane = wp.rank();
  int top = 0;
  if (lane == 0) { stk[0] = l; stk[1] = h; stk[2] = d; }
  ++top;
  wp.sync();
  while (top > 0) {
    --top;
    const int sl = stk[3 * top], sh = stk[3 * top + 1], sd = stk[3 * top + 2];
    wp.sync();
    if (sd == 0) {
      if (lane == 0) {
        ox_heap_sort(zk, sq, sl, sh);
        if (stats) atomicAdd(stats + 1, 1ull);
      }
      wp.sync();
      continue;
    }
    const int cut = ox_partition(wp, zk, sq, ix + sl, ix + n + sl, sl, sh);
    if (sh - cut > OX_THRESHOLD) {
      if (lane == 0) { stk[3 * top] = cut; stk[3 * top + 1] = sh; stk[3 * top + 2] = sd - 1; }
      ++top;
    }
    if (cut - sl > OX_THRESHOLD) {
      if (lane == 0) { stk[3 * top] = sl; stk[3 * top + 1] = cut; stk[3 * top + 2] = sd - 1; }
      ++top;
    }
    wp.sync();
  }
}

__device__ __forceinline__ int ox_find(const int* idx, int n, int v) {   // position of point index v in the bin (ascending indices)
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (idx[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Steps 1 to 3 of one patch by one team; loop(zk, sq, ix) runs the introsort loop of step 2. ws: ox_ws_words(n) words.
template <class Team, class Loop>
__device__ __forceinline__ void ox_patch(const Team& tm, const float4* P, const unsigned char* L, int* out, int n, unsigned* ws, int* stk,
                                         unsigned long long* stats, Loop loop) {
  float* zk = reinterpret_cast<float*>(ws);
  int* sq = reinterpret_cast<int*>(ws + n);
  int* ix = reinterpret_cast<int*>(ws + 2 * n);
  bool flag = false;
  for (int i = tm.rank(); i < n; i += Team::size) {
    const float4 q = P[i];
    zk[i] = q.z;
    sq[i] = __float_as_int(q.w);
    flag |= q.z != q.z;
  }
  const bool nan = tm.any(flag);
  if (!nan) {
    for (int k = tm.rank(); k < n; k += Team::size) ix[k] = ox_find(sq, n, out[k]);
    tm.sync();
    flag = false;
    for (int k = tm.rank(); k + 1 < n; k += Team::size) {
      const int a = ix[k], b = ix[k + 1];
      flag |= L[a] == L[b] && zk[a] == zk[b];
    }
    if (!tm.any(flag)) return;
  }
  for (int i = tm.rank(); i < n; i += Team::size) sq[i] = i;
  tm.sync();
  if (tm.rank() == 0 && stats) atomicAdd(stats + (nan ? 2 : 0), 1ull);
  if (nan) {
    if (tm.rank() == 0) ox_std_sort_serial(zk, sq, n, stk, stats);
    tm.sync();
  } else if (n > OX_THRESHOLD) {
    loop(zk, sq, ix);
  }
  // (group, z, q), or (group, q) where the sequence is std::sort's output already
  unsigned long long* key = reinterpret_cast<unsigned long long*>(ws + 2 * n);
  for (int q = tm.rank(); q < n; q += Team::size) {
    const unsigned char lab = L[sq[q]];
    if (nan) {
      const unsigned grp = lab == PW_LABEL_GROUND ? 0u : (lab == PW_LABEL_REJECT ? 9u : (unsigned) lab);
      key[q] = ((unsigned long long) grp << 56) | (unsigned) q;
    } else {
      key[q] = order_sort_key(zk[q], lab, (unsigned) q);
    }
  }
  tm.sync();
  for (int k = 2; (k >> 1) < n; k <<= 1) {   // bitonic, every compare-exchange ascending: the virtual padding above n never moves
    for (int j = k - 1; j > 0; j = (j == k - 1) ? (k >> 2) : (j >> 1)) {
      for (int i = tm.rank(); i < n; i += Team::size) {
        const int l = i ^ j;
        if (l > i && l < n) {
          const unsigned long long a = key[i], b = key[l];
          if (a > b) { key[i] = b; key[l] = a; }
        }
      }
      tm.sync();
    }
  }
  for (int k = tm.rank(); k < n; k += Team::size) out[k] = __float_as_int(P[sq[(int) (key[k] & 0xffffffull)]].w);
  tm.sync();
}

// Classes L1, L2, L3 and X (queue CLS): one warp per patch as for classes M and S, persistent, after k_order_cta<., CLS> on the
// same stream; the workspace in the global scratch xws, the warp's stack in shared memory. stats may be null.
template <int CLS>
__global__ void __launch_bounds__(OX_WARP_THREADS, 1) k_order_exact_big(const float4* __restrict__ sorted, WorkQueues wq, int* __restrict__ head, int* __restrict__ part,
                                                                     unsigned* __restrict__ xws, unsigned long long* __restrict__ stats) {
  __shared__ int s_stk[OX_WARP_THREADS / 32][OX_STACK * 3];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int* stk = s_stk[w];
  const OxWarp wp;
  const int total = wq.count[CLS];
  for (;;) {
    int t = 0;
    if (lane == 0) t = atomicAdd(head, 1);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= total) return;
    const int4 wi = wq.items[CLS][t];
    const int n = wi.y;
    const long long start = work_item_start(wi);
    unsigned* ws = xws + OX_X_WORDS * start;
    ox_patch(wp, sorted + start, wq.labels + start, part + start, n, ws, stk, stats, [=](float* zk, int* sq, int* ix) {
      ox_warp_loop(zk, sq, ix, n, stk, 0, n, 2 * (31 - __clz(n)), stats);
    });
  }
}

// Classes M and S: one warp per patch, the whole patch in the warp's share of shared memory, after k_order_warp.
__global__ void __launch_bounds__(OX_WARP_THREADS) k_order_exact_warp(const float4* __restrict__ sorted, WorkQueues wq, int* __restrict__ head, int* __restrict__ part,
                                                                      unsigned long long* __restrict__ stats) {
  PW_DYN_SHARED(unsigned, s_all);   // per warp: ox_ws_words(CLS_M_MAX) words of workspace, then OX_STACK * 3 of stack
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned* ws = s_all + (size_t) w * (ox_ws_words(CLS_M_MAX) + 3 * OX_STACK);
  int* stk = reinterpret_cast<int*>(ws + ox_ws_words(CLS_M_MAX));
  const OxWarp wp;
  const int n_m = wq.count[1], total = n_m + wq.count[0];
  for (;;) {
    int t = 0;
    if (lane == 0) t = atomicAdd(head, 1);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= total) return;
    const int4 wi = t < n_m ? wq.items[1][t] : wq.items[0][t - n_m];
    const int n = wi.y;
    const long long start = work_item_start(wi);
    ox_patch(wp, sorted + start, wq.labels + start, part + start, n, ws, stk, stats, [=](float* zk, int* sq, int* ix) {
      ox_warp_loop(zk, sq, ix, n, stk, 0, n, 2 * (31 - __clz(n)), stats);
    });
  }
}

}  // namespace pwpp

// pwpp_records.cuh — sensor point records of any PointCloud2 layout -> the engine's packed float4 {x, y, z, intensity} points
// (pwpp_estimate_host_records / pwpp_estimate_device_records, include/pwpp.h).
//
// One launch unpacks every frame of a launch range: blockIdx.y is the frame, blockIdx.x a tile of its records. The pass is
// memory-bound (point_step bytes read and 16 written per point), so a CTA first stages its tile's contiguous byte range
// [src + i0 * step, src + i1 * step) in shared memory: 16-byte vector loads for the 16-byte-aligned body of the range, byte loads
// for the unaligned head and tail (at most 15 bytes each), so a 22-byte record still reads HBM in whole sectors, and no byte
// outside the frame is touched (a caller's frame may be a view that ends anywhere). Every thread then assembles its records'
// fields from aligned shared-memory words (funnel shifts: any field alignment), converts them to float with round-to-nearest
// and stores one float4 per point. The datatype of a field is uniform per frame, hence per CTA: its switch does not diverge.
#pragma once
#include "pwpp_common.cuh"
#include "pwpp.h"

namespace pwpp {

// per-frame entry of the call's record table (uploaded with the frame tables): where frame f's records are and how to read them
struct RecordFrame {
  const unsigned char* src;   // first byte of record 0 (device memory: the caller's buffer or the ctx's upload buffer)
  int step;                   // point_step, 1..PWPP_MAX_POINT_STEP
  int off[4];                 // byte offsets of x, y, z, intensity inside a record
  int type[4];                // PWPP_FIELD_*; type[3] = 0: the frame has no intensity field (NaN intensity)
  int pad;
};
static_assert(sizeof(RecordFrame) == 48, "RecordFrame is uploaded as a 48-byte record");

constexpr int REC_THREADS = 256;
constexpr int REC_TILE_BYTES = 16384;    // bytes of records one CTA stages (whole records)
constexpr int REC_MAX_TILE_PTS = 1024;
// shared memory: the tile, the up to 15 bytes below its first 16-byte boundary, and room for the word reads of the last field
constexpr int REC_SMEM_WORDS = (REC_TILE_BYTES + 32) / 4;

// records per CTA for a record size: 1024 for steps up to 16, 16 at the largest step
__host__ __device__ inline int rec_tile_pts(int step) {
  const int t = REC_TILE_BYTES / step;
  return t < REC_MAX_TILE_PTS ? t : REC_MAX_TILE_PTS;
}

#if defined(PWPP_SIMT_EMU)
inline float rec_i2f(int v) { return (float) v; }                 // the host's conversions round to nearest, as numpy does
inline float rec_u2f(unsigned v) { return (float) v; }
inline float rec_d2f(double v) { return (float) v; }
inline double rec_lohi2d(unsigned lo, unsigned hi) { const unsigned long long b = ((unsigned long long) hi << 32) | lo; double d; std::memcpy(&d, &b, 8); return d; }
inline void rec_ld16(void* dst, const unsigned char* p) { std::memcpy(dst, p, 16); }   // (the SIMT stand-in: a plain load)
#else
__device__ __forceinline__ float rec_i2f(int v) { return __int2float_rn(v); }
__device__ __forceinline__ float rec_u2f(unsigned v) { return __uint2float_rn(v); }
__device__ __forceinline__ float rec_d2f(double v) { return __double2float_rn(v); }
__device__ __forceinline__ double rec_lohi2d(unsigned lo, unsigned hi) { return __hiloint2double((int) hi, (int) lo); }
// read-once records: 16-byte load that does not allocate in L1
__device__ __forceinline__ void rec_ld16(void* dst, const unsigned char* p) {
  uint4 v;
  asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  *reinterpret_cast<uint4*>(dst) = v;
}
#endif

// the 4 bytes starting at byte b of the staged words, any alignment (little-endian)
__device__ __forceinline__ unsigned rec_word(const unsigned* s, int b) {
  const unsigned lo = s[b >> 2], hi = s[(b >> 2) + 1];
  return (unsigned) ((((unsigned long long) hi << 32) | lo) >> ((b & 3) * 8));
}

// FLOAT64 -> float with round-to-nearest-even; a NaN keeps its sign and the top 22 payload bits and becomes quiet (what x86's
// conversion, and so numpy's astype(np.float32), produces; the H100's instruction alone gave the same bits on every NaN tested: the branch makes it a rule)
__device__ __forceinline__ float rec_f64(unsigned lo, unsigned hi) {
  const double d = rec_lohi2d(lo, hi);
  if (d != d) return __uint_as_float((hi & 0x80000000u) | 0x7fc00000u | ((hi & 0x000fffffu) << 3) | (lo >> 29));
  return rec_d2f(d);
}

__device__ __forceinline__ float rec_field(const unsigned* s, int b, int type) {
  const unsigned w = rec_word(s, b);
  switch (type) {
    case PWPP_FIELD_INT8: return rec_i2f((int) (signed char) (w & 0xffu));
    case PWPP_FIELD_UINT8: return rec_u2f(w & 0xffu);
    case PWPP_FIELD_INT16: return rec_i2f((int) (short) (w & 0xffffu));
    case PWPP_FIELD_UINT16: return rec_u2f(w & 0xffffu);
    case PWPP_FIELD_INT32: return rec_i2f((int) w);
    case PWPP_FIELD_UINT32: return rec_u2f(w);
    case PWPP_FIELD_FLOAT32: return __uint_as_float(w);
    case PWPP_FIELD_FLOAT64: return rec_f64(w, rec_word(s, b + 4));
    default: return __uint_as_float(0x7fc00000u);   // no intensity field: a NaN fails every RNR test (rnr_hit)
  }
}

// frame f = blockIdx.y of the range: records tile blockIdx.x -> dst[pt_off[f] + i]. pt_off holds absolute positions (the
// call's frame table offset to the range's first frame).
__global__ void __launch_bounds__(REC_THREADS) k_unpack_records(const RecordFrame* __restrict__ recs, const long long* __restrict__ pt_off,
                                                                 float4* __restrict__ dst) {
  __shared__ __align__(16) unsigned s_w[REC_SMEM_WORDS];
  const int f = blockIdx.y, tid = threadIdx.x;
  const RecordFrame R = recs[f];
  const long long p0 = pt_off[f];
  const long long n = pt_off[f + 1] - p0;
  const int tp = rec_tile_pts(R.step);
  const long long i0 = (long long) blockIdx.x * tp;
  if (i0 >= n) return;
  const int cnt = (int) (n - i0 < tp ? n - i0 : tp);
  const unsigned char* a = R.src + i0 * R.step;                 // the tile's bytes [a, b)
  const unsigned char* b = a + (size_t) cnt * R.step;
  const unsigned char* a_floor = (const unsigned char*) ((uintptr_t) a & ~(uintptr_t) 15);   // shared word 0 holds this address
  const unsigned char* a16 = (const unsigned char*) (((uintptr_t) a + 15) & ~(uintptr_t) 15);
  const unsigned char* b16 = (const unsigned char*) ((uintptr_t) b & ~(uintptr_t) 15);
  unsigned char* s_b = reinterpret_cast<unsigned char*>(s_w);
  if (a16 < b16) {
    const int nvec = (int) ((b16 - a16) >> 4), vbase = (int) (a16 - a_floor);
#pragma unroll 4
    for (int k = tid; k < nvec; k += REC_THREADS) rec_ld16(s_b + vbase + 16 * k, a16 + 16 * k);
    const int head = (int) (a16 - a), tail = (int) (b - b16);
    if (tid < head) s_b[(a - a_floor) + tid] = a[tid];
    else if (tid >= 16 && tid < 16 + tail) s_b[(b16 - a_floor) + (tid - 16)] = b16[tid - 16];
  } else {
    for (int k = tid; k < (int) (b - a); k += REC_THREADS) s_b[(a - a_floor) + k] = a[k];
  }
  __syncthreads();
  const int r0 = (int) (a - a_floor);
  float4* out = dst + p0 + i0;
  for (int i = tid; i < cnt; i += REC_THREADS) {
    const int r = r0 + i * R.step;
    out[i] = make_float4(rec_field(s_w, r + R.off[0], R.type[0]), rec_field(s_w, r + R.off[1], R.type[1]), rec_field(s_w, r + R.off[2], R.type[2]),
                         rec_field(s_w, r + R.off[3], R.type[3]));
  }
}

// Entry of the record table for a frame of this (validated) layout whose records start at src (device memory).
inline RecordFrame record_frame(const pwpp_point_layout& L, const void* src) {
  RecordFrame r{};
  r.src = static_cast<const unsigned char*>(src);
  r.step = L.point_step;
  for (int c = 0; c < 4; ++c) { r.off[c] = L.offset[c]; r.type[c] = L.datatype[c]; }
  if (L.offset[3] < 0) { r.off[3] = 0; r.type[3] = 0; }   // no intensity field: the kernel writes NaN
  return r;
}

// ---- bound calls (pwpp_bind_call / pwpp_run_bound_call): the frame tables from sizes that live on the device ---------------
//
// k_bound_table is one CTA. Thread t owns a contiguous slice of ceil(nf / BT_THREADS) frames: it accepts every count of its
// slice (0 <= counts[f] <= max_n[f]; any other count makes an empty frame and sets status[f]), sums the accepted sizes and
// their chunks, a warp-shuffle scan and a scan of the warp totals give every slice its start, and a second pass writes the
// slice's entries: pt_off (int64 exclusive scan of the accepted counts, nf + 1 entries), chunk_off (scan of ceil(n / CHUNK_PTS),
// nf + 1), status, and the bound call's own stream and set tables copied into the call tables, which direct calls between two
// runs overwrite. The bind checked that the chunks of the capacities fit an int, so the accepted ones do too.
//
// With per-frame actions (pwpp_bind_call_actions) the same kernel, k_bound_table_actions, also reads every frame's action once
// (actions[f], the caller's device array) into the ctx's copy act[f], which every later kernel of the run reads. A frame that is
// not PWPP_FRAME_RUN or PWPP_FRAME_RESET is skipped: its count is not read, it runs as an empty frame, status[f] is
// PWPP_FRAME_SKIPPED (PWPP_ACTION_INVALID for an unknown value), and stream[f] is its scratch slot scratch[f], so k_gle writes
// the empty frame's update there and the real stream is never touched. A RESET frame whose stream has no frame in an earlier
// run (dep[f] == 0) gets its stream's constructor state here, before any run; the others are reset by k_bound_reset right
// before their run.
//
// With scan rings (pwpp_bind_call_rings), k_bound_table_rings / k_bound_table_rings_actions also pick every frame's address:
// a frame that runs reads its slot s = slots[f] once into the ctx's copy slot[f] (-1 for a skipped frame), takes its count
// from its ring's counts[s] and writes the run's record table entry brun[f] = the bound entry brec[f] with src = base +
// s * stride. A slot outside [0, num_slots) makes an empty frame with status PWPP_SLOT_OUT_OF_RANGE; skipped frames and those
// keep src = base with n = 0, so nothing is read. The unpack and the record gather of the run read brun.
//
// With a packed buffer (pwpp_bind_call_packed), k_bound_table_packed / k_bound_table_packed_actions pick every frame's records
// from the caller's device offsets: a frame that runs reads lo = offsets[f] and hi = offsets[f + 1]; offsets outside
// 0 <= lo <= hi <= capacity make an empty frame with status PWPP_OFFSETS_OUT_OF_RANGE, a count hi - lo above max_n[f] one with
// PWPP_COUNT_OUT_OF_RANGE, and an accepted frame's entry brun[f] is brec[f] with src = base + lo * step. Every other frame keeps
// src = base with n = 0. A skipped frame reads neither offset.
//
// With a stream table (pwpp_bind_stream_table), k_bound_table_streams / _rings_streams / _packed_streams take every frame's
// stream from the caller's device array instead of the bound table: read once into the ctx's copy (bt_stream_verdicts), the
// set from the device map set_of, holes, out-of-range ids and duplicates inside a run skipped to the scratch slot as an action
// SKIP is. They always take the actions form (A.actions may be NULL: every frame RUN).
constexpr int BT_THREADS = 1024;

// The CTA-wide scan of the one-CTA table kernels (bound_table_body, k_bound_xyz_offsets): each of the BT_THREADS threads (lane,
// warp) brings the sums own_a, own_b of its slice of frames and gets back in a, b their exclusive prefix sums, the start of its
// slice: a warp-shuffle scan, then one of the warp totals in s_a, s_b (BT_THREADS / 32 entries each).
template <typename A, typename B>
__device__ __forceinline__ void bt_scan_slices(int lane, int warp, A own_a, B own_b, A& a, B& b, A* s_a, B* s_b) {
  A pa = own_a;   // inclusive scan over the warp's slices
  B pb = own_b;
  for (int d = 1; d < 32; d <<= 1) {
    const A p = __shfl_up_sync(0xffffffffu, pa, d);
    const B q = __shfl_up_sync(0xffffffffu, pb, d);
    if (lane >= d) { pa += p; pb += q; }
  }
  if (lane == 31) { s_a[warp] = pa; s_b[warp] = pb; }
  __syncthreads();
  if (warp == 0) {   // inclusive scan of the warp totals
    A wa = s_a[lane];
    B wb = s_b[lane];
    for (int d = 1; d < 32; d <<= 1) {
      const A p = __shfl_up_sync(0xffffffffu, wa, d);
      const B q = __shfl_up_sync(0xffffffffu, wb, d);
      if (lane >= d) { wa += p; wb += q; }
    }
    s_a[lane] = wa;
    s_b[lane] = wb;
  }
  __syncthreads();
  a = (warp > 0 ? s_a[warp - 1] : 0) + pa - own_a;
  b = (warp > 0 ? s_b[warp - 1] : 0) + pb - own_b;
}

struct BoundActions {
  const int* actions;            // the caller's device actions [nf]
  int* act;                      // the ctx's copy [nf]
  const int* scratch;            // scratch slot of every frame [nf]
  const int* dep;                // 1: the frame's stream has a frame in an earlier run [nf]
  const StreamState* init;       // constructor state of every stream
  StreamState* states;
};

// frame f's action from the caller's array, copied for the later kernels of the run (actions of a bound call without them: RUN)
template <bool Actions>
__device__ __forceinline__ int bt_action(const BoundActions& A, int f) {
  if (!Actions) return PWPP_FRAME_RUN;
  const int a = A.actions[f];
  A.act[f] = a;
  return a;
}
__device__ __forceinline__ bool bt_runs(int a) { return a == PWPP_FRAME_RUN || a == PWPP_FRAME_RESET; }

// one frame's ring (uploaded at bind time, next to max_n and the stream table)
struct BoundRing {
  const long long* counts;       // the caller's device counts [num_slots]
  long long stride;              // bytes from slot s to slot s + 1
  int num_slots;
  int pad;
};
static_assert(sizeof(BoundRing) == 24, "BoundRing is uploaded as a 24-byte record");

struct BoundRings {
  const int* slots;              // the caller's device slots [nf]
  int* slot;                     // the ctx's copy [nf]: the slot each frame read, -1 for a skipped frame
  const BoundRing* ring;         // [nf]
  const RecordFrame* brec;       // the bound record table (src: slot 0)
  RecordFrame* brun;             // the run's record table
};

__device__ __forceinline__ bool bt_slot_ok(int s, const BoundRing& R) { return s >= 0 && s < R.num_slots; }

// frame f's count for the first pass: counts[f], or with rings its slot's count (the slot read once and copied; -1, an empty
// frame, for a slot out of range)
template <bool Rings>
__device__ __forceinline__ long long bt_count(const long long* __restrict__ counts, const BoundRings& G, int f) {
  if (!Rings) return counts[f];
  const int s = G.slots[f];
  G.slot[f] = s;
  const BoundRing R = G.ring[f];
  return bt_slot_ok(s, R) ? R.counts[s] : -1;
}

// the packed buffer of a bound call (pwpp_bind_call_packed)
struct BoundPacked {
  const long long* offsets;      // the caller's device offsets [nf + 1]
  long long capacity;            // records at the bound base
  const RecordFrame* brec;       // the bound record table (src: base)
  RecordFrame* brun;             // the run's record table
};

__device__ __forceinline__ bool bt_offsets_ok(long long lo, long long hi, long long capacity) { return lo >= 0 && hi >= lo && hi <= capacity; }

// frame f's count from its two offsets, -1 (an empty frame) for offsets out of range
__device__ __forceinline__ long long bt_packed_count(const BoundPacked& P, int f) {
  const long long lo = P.offsets[f], hi = P.offsets[f + 1];
  return bt_offsets_ok(lo, hi, P.capacity) ? hi - lo : -1;
}

// the stream table of a bound call (pwpp_bind_stream_table)
struct BoundStreams {
  const int* streams;            // the caller's device streams [nf]
  int* read;                     // the ctx's copy [nf]: what every frame read, invalid values included
  int* claim;                    // [num_streams] duplicate claims, -1 between runs
  const int* set_of;             // [num_streams] parameter set of every stream
  const int* runs;               // [nruns + 1] the bound runs
  int nruns, num_streams;
};

// With a stream table, before the count pass: every frame's action (NULL actions: RUN) and stream, read once and copied, and a
// first verdict in status[f] that the later passes of the same thread read back: the action's skip status, then
// PWPP_FRAME_SKIPPED for a hole (s < 0), PWPP_STREAM_OUT_OF_RANGE, or, run by run, PWPP_STREAM_DUPLICATE for a frame that would
// run but whose stream an earlier frame of the run claimed. A claim is an atomicMax of INT_MAX - f on claim[s]: the lowest
// position wins, and the -1 of an unclaimed entry is below every key. The claims are put back to -1 before the next run.
// A frame rejected by its stream gets PWPP_FRAME_SKIP in the action copy, so that k_bound_reset leaves its stream alone.
__device__ __forceinline__ void bt_stream_verdicts(int f0, int f1, const BoundActions& A, const BoundStreams& T, int* __restrict__ status) {
  for (int f = f0; f < f1; ++f) {
    const int a = A.actions ? A.actions[f] : PWPP_FRAME_RUN;
    const int s = T.streams[f];
    T.read[f] = s;
    int v = 0;
    if (!bt_runs(a)) v = a == PWPP_FRAME_SKIP ? PWPP_FRAME_SKIPPED : PWPP_ACTION_INVALID;
    else if (s < 0) v = PWPP_FRAME_SKIPPED;
    else if (s >= T.num_streams) v = PWPP_STREAM_OUT_OF_RANGE;
    if (A.act) A.act[f] = (v != 0 && bt_runs(a)) ? PWPP_FRAME_SKIP : a;
    status[f] = v;
  }
  for (int r = 0; r < T.nruns; ++r) {   // every thread takes part in every run's barriers; its slice may span several runs
    const int r0 = max(f0, T.runs[r]), r1 = min(f1, T.runs[r + 1]);
    for (int f = r0; f < r1; ++f)
      if (status[f] == 0) atomicMax(&T.claim[T.read[f]], 0x7fffffff - f);
    __syncthreads();
    for (int f = r0; f < r1; ++f) {
      if (status[f] != 0) continue;
      if (*(volatile const int*) &T.claim[T.read[f]] != 0x7fffffff - f) {   // volatile: the claims changed since any earlier load
        status[f] = PWPP_STREAM_DUPLICATE;
        if (A.act) A.act[f] = PWPP_FRAME_SKIP;
      }
    }
    __syncthreads();
    for (int f = r0; f < r1; ++f)
      if (status[f] == 0) T.claim[T.read[f]] = -1;   // the winner, the one frame of the run left on its stream
    __syncthreads();
  }
}

template <bool Actions, bool Rings = false, bool Packed = false, bool Streams = false>
__device__ __forceinline__ void bound_table_body(int nf, const long long* __restrict__ counts, const long long* __restrict__ max_n,
                                                 const int* __restrict__ b_stream, const int* __restrict__ b_pset, long long* __restrict__ pt_off,
                                                 int* __restrict__ chunk_off, int* __restrict__ stream, int* __restrict__ pset,
                                                 int* __restrict__ status, const BoundActions& A, long long* s_pts, int* s_chk,
                                                 const BoundRings& G = BoundRings{}, const BoundPacked& P = BoundPacked{},
                                                 const BoundStreams& T = BoundStreams{}) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (nf + BT_THREADS - 1) / BT_THREADS;
  const int f0 = tid * per < nf ? tid * per : nf;
  const int f1 = f0 + per < nf ? f0 + per : nf;
  long long own_pts = 0;
  int own_chk = 0;
  if (Streams) bt_stream_verdicts(f0, f1, A, T, status);
  for (int f = f0; f < f1; ++f) {
    long long n = 0;
    if (Streams ? status[f] == 0 : bt_runs(bt_action<Actions>(A, f))) {
      const long long c = Packed ? bt_packed_count(P, f) : bt_count<Rings>(counts, G, f);
      n = (c >= 0 && c <= max_n[f]) ? c : 0;
    } else if (Rings) {
      G.slot[f] = -1;
    }
    own_pts += n;
    own_chk += (int) ((n + CHUNK_PTS - 1) / CHUNK_PTS);
  }
  long long p;   // the start of the slice
  int q;
  bt_scan_slices(lane, warp, own_pts, own_chk, p, q, s_pts, s_chk);
  for (int f = f0; f < f1; ++f) {
    int sf = 0, ps = 0;   // with a stream table: the frame's stream and set
    if (Streams) {
      sf = T.read[f];   // this thread's own copies from the first pass
      const int v = status[f];
      if (v != 0) {
        pt_off[f] = p;
        chunk_off[f] = q;
        stream[f] = A.scratch[f];
        pset[f] = sf >= 0 && sf < T.num_streams ? T.set_of[sf] : b_pset[f];
        if (Rings) G.brun[f] = G.brec[f];
        if (Packed) P.brun[f] = P.brec[f];
        continue;
      }
      ps = T.set_of[sf];
      if (A.act && A.act[f] == PWPP_FRAME_RESET && !A.dep[f]) A.states[sf] = A.init[sf];
    }
    if (Actions && !Streams) {
      const int a = A.act[f];   // this thread's own copy from the first pass
      if (!bt_runs(a)) {
        pt_off[f] = p;
        chunk_off[f] = q;
        status[f] = a == PWPP_FRAME_SKIP ? PWPP_FRAME_SKIPPED : PWPP_ACTION_INVALID;
        stream[f] = A.scratch[f];
        pset[f] = b_pset[f];
        if (Rings) G.brun[f] = G.brec[f];
        if (Packed) P.brun[f] = P.brec[f];
        continue;
      }
      if (a == PWPP_FRAME_RESET && !A.dep[f]) A.states[b_stream[f]] = A.init[b_stream[f]];
    }
    long long c;
    int bad = PWPP_COUNT_OUT_OF_RANGE;
    if (Rings) {
      const int s = G.slot[f];   // this thread's own copy from the first pass
      const BoundRing R = G.ring[f];
      RecordFrame r = G.brec[f];
      if (bt_slot_ok(s, R)) {
        c = R.counts[s];
        r.src += (long long) s * R.stride;
      } else {
        c = -1;
        bad = PWPP_SLOT_OUT_OF_RANGE;
      }
      G.brun[f] = r;
    } else if (Packed) {
      const long long lo = P.offsets[f], hi = P.offsets[f + 1];
      if (bt_offsets_ok(lo, hi, P.capacity)) {
        c = hi - lo;
      } else {
        c = -1;
        bad = PWPP_OFFSETS_OUT_OF_RANGE;
      }
      RecordFrame r = P.brec[f];
      if (c >= 0 && c <= max_n[f]) r.src += lo * r.step;
      P.brun[f] = r;
    } else {
      c = counts[f];
    }
    const bool ok = c >= 0 && c <= max_n[f];
    const long long n = ok ? c : 0;
    pt_off[f] = p;
    chunk_off[f] = q;
    status[f] = ok ? 0 : bad;
    stream[f] = Streams ? sf : b_stream[f];
    pset[f] = Streams ? ps : b_pset[f];
    p += n;
    q += (int) ((n + CHUNK_PTS - 1) / CHUNK_PTS);
  }
  if (tid == BT_THREADS - 1) { pt_off[nf] = p; chunk_off[nf] = q; }   // the last slice ends at the totals
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table(int nf, const long long* __restrict__ counts, const long long* __restrict__ max_n,
                                                            const int* __restrict__ b_stream, const int* __restrict__ b_pset,
                                                            long long* __restrict__ pt_off, int* __restrict__ chunk_off, int* __restrict__ stream,
                                                            int* __restrict__ pset, int* __restrict__ status) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<false>(nf, counts, max_n, b_stream, b_pset, pt_off, chunk_off, stream, pset, status, BoundActions{}, s_pts, s_chk);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_actions(int nf, const long long* __restrict__ counts, const long long* __restrict__ max_n,
                                                                    const int* __restrict__ b_stream, const int* __restrict__ b_pset,
                                                                    long long* __restrict__ pt_off, int* __restrict__ chunk_off, int* __restrict__ stream,
                                                                    int* __restrict__ pset, int* __restrict__ status, const BoundActions A) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<true>(nf, counts, max_n, b_stream, b_pset, pt_off, chunk_off, stream, pset, status, A, s_pts, s_chk);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_rings(int nf, const long long* __restrict__ max_n, const int* __restrict__ b_stream,
                                                                  const int* __restrict__ b_pset, long long* __restrict__ pt_off,
                                                                  int* __restrict__ chunk_off, int* __restrict__ stream, int* __restrict__ pset,
                                                                  int* __restrict__ status, const BoundRings G) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<false, true>(nf, nullptr, max_n, b_stream, b_pset, pt_off, chunk_off, stream, pset, status, BoundActions{}, s_pts, s_chk, G);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_rings_actions(int nf, const long long* __restrict__ max_n, const int* __restrict__ b_stream,
                                                                          const int* __restrict__ b_pset, long long* __restrict__ pt_off,
                                                                          int* __restrict__ chunk_off, int* __restrict__ stream, int* __restrict__ pset,
                                                                          int* __restrict__ status, const BoundActions A, const BoundRings G) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<true, true>(nf, nullptr, max_n, b_stream, b_pset, pt_off, chunk_off, stream, pset, status, A, s_pts, s_chk, G);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_packed(int nf, const long long* __restrict__ max_n, const int* __restrict__ b_stream,
                                                                   const int* __restrict__ b_pset, long long* __restrict__ pt_off,
                                                                   int* __restrict__ chunk_off, int* __restrict__ stream, int* __restrict__ pset,
                                                                   int* __restrict__ status, const BoundPacked P) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<false, false, true>(nf, nullptr, max_n, b_stream, b_pset, pt_off, chunk_off, stream, pset, status, BoundActions{}, s_pts, s_chk,
                                       BoundRings{}, P);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_packed_actions(int nf, const long long* __restrict__ max_n, const int* __restrict__ b_stream,
                                                                           const int* __restrict__ b_pset, long long* __restrict__ pt_off,
                                                                           int* __restrict__ chunk_off, int* __restrict__ stream, int* __restrict__ pset,
                                                                           int* __restrict__ status, const BoundActions A, const BoundPacked P) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<true, false, true>(nf, nullptr, max_n, b_stream, b_pset, pt_off, chunk_off, stream, pset, status, A, s_pts, s_chk, BoundRings{}, P);
}

// The three sources with a stream table (pwpp_bind_stream_table), with or without actions (A.actions NULL: every frame RUN,
// A.act NULL: no copy, no reset).
__global__ void __launch_bounds__(BT_THREADS) k_bound_table_streams(int nf, const long long* __restrict__ counts, const long long* __restrict__ max_n,
                                                                    const int* __restrict__ b_pset, long long* __restrict__ pt_off,
                                                                    int* __restrict__ chunk_off, int* __restrict__ stream, int* __restrict__ pset,
                                                                    int* __restrict__ status, const BoundActions A, const BoundStreams T) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<true, false, false, true>(nf, counts, max_n, nullptr, b_pset, pt_off, chunk_off, stream, pset, status, A, s_pts, s_chk,
                                             BoundRings{}, BoundPacked{}, T);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_rings_streams(int nf, const long long* __restrict__ max_n, const int* __restrict__ b_pset,
                                                                          long long* __restrict__ pt_off, int* __restrict__ chunk_off,
                                                                          int* __restrict__ stream, int* __restrict__ pset, int* __restrict__ status,
                                                                          const BoundActions A, const BoundRings G, const BoundStreams T) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<true, true, false, true>(nf, nullptr, max_n, nullptr, b_pset, pt_off, chunk_off, stream, pset, status, A, s_pts, s_chk, G,
                                            BoundPacked{}, T);
}

__global__ void __launch_bounds__(BT_THREADS) k_bound_table_packed_streams(int nf, const long long* __restrict__ max_n, const int* __restrict__ b_pset,
                                                                           long long* __restrict__ pt_off, int* __restrict__ chunk_off,
                                                                           int* __restrict__ stream, int* __restrict__ pset, int* __restrict__ status,
                                                                           const BoundActions A, const BoundPacked P, const BoundStreams T) {
  __shared__ long long s_pts[BT_THREADS / 32];
  __shared__ int s_chk[BT_THREADS / 32];
  bound_table_body<true, false, true, true>(nf, nullptr, max_n, nullptr, b_pset, pt_off, chunk_off, stream, pset, status, A, s_pts, s_chk,
                                            BoundRings{}, P, T);
}

// k_bound_reset: one CTA before run [f0, f1) of a bound call with actions, launched only for runs that hold a frame whose stream
// has a frame in an earlier run. Every such frame whose action (the run's copy, act) is PWPP_FRAME_RESET restores its stream's
// constructor state: the StreamState only, as pwpp_reset_stream (the history sizes live in it). The run's streams are
// pairwise distinct, so no two threads write one state. With a stream table it runs before every run after the first, over the
// run's copy of the streams (every dep is 1 there; a frame its stream rejected has SKIP in the action copy).
constexpr int BR_THREADS = 128;

__global__ void __launch_bounds__(BR_THREADS) k_bound_reset(int f0, int f1, const int* __restrict__ act, const int* __restrict__ dep,
                                                            const int* __restrict__ b_stream, const StreamState* __restrict__ init,
                                                            StreamState* __restrict__ states) {
  for (int f = f0 + (int) threadIdx.x; f < f1; f += BR_THREADS)
    if (dep[f] && act[f] == PWPP_FRAME_RESET) states[b_stream[f]] = init[b_stream[f]];
}

// grid.x of a launch over frames with these sizes and steps
inline long long rec_grid_x(const long long* pt_off, const RecordFrame* recs, int nf) {
  long long gx = 0;
  for (int f = 0; f < nf; ++f) {
    const int tp = rec_tile_pts(recs[f].step);
    const long long t = (pt_off[f + 1] - pt_off[f] + tp - 1) / tp;
    gx = t > gx ? t : gx;
  }
  return gx;
}

// ---- the way back: the segmented lists as whole records of each frame's own layout (pwpp_*_record_results) ----------------
//
// k_gather_records writes, for every frame f of a call, output record k (0 <= k < ng + nn) = input record idx[pt_off[f] + k],
// byte for byte, to dst + rec_off[f] + k * step: the ground list, then the non-ground list, as k_emit left them. The dropped
// count (ng + nn = n - dropped) comes from the device (the call's count row), so the host sizes the grid from n[f] alone and
// CTAs past ng + nn return at once. A CTA assembles a tile of whole output records (rec_tile_pts) in shared memory, laid out at the
// tile's own distance from a 16-byte boundary of dst: every thread builds aligned shared words from the frame's records with
// aligned 4-byte loads (a 64-bit shift re-aligns them: a funnel shift), byte loads where a word would reach outside the frame,
// then the tile goes out with 16-byte stores for its aligned body and byte stores for its head and tail (at most 15 bytes each).
// The sources of a tile are scattered and each word's address depends on a shared-memory load of its record's index, so a
// thread issues the loads of REC_GW words before it assembles any of them: memory-level parallelism, not bandwidth, is what
// a gather of 4-byte words runs out of first.
// No byte outside [src, src + n * step) is read and none outside [rec_off[f], rec_off[f] + (ng + nn) * step) is written.

#if defined(PWPP_SIMT_EMU)
inline unsigned rec_ld4(const unsigned char* p) { unsigned v; std::memcpy(&v, p, 4); return v; }
inline void rec_st16(unsigned char* p, const void* src) { std::memcpy(p, src, 16); }
#else
__device__ __forceinline__ unsigned rec_ld4(const unsigned char* p) { return __ldg(reinterpret_cast<const unsigned*>(p)); }
// written once, read by the caller's D2H or kernels: a streaming store
__device__ __forceinline__ void rec_st16(unsigned char* p, const void* src) { __stcs(reinterpret_cast<uint4*>(p), *reinterpret_cast<const uint4*>(src)); }
#endif

constexpr int REC_GW = 4;   // words a thread of k_gather_records has in flight (two aligned loads per record piece)

// the 4 bytes at p of the frame, one at a time; bytes at or beyond hi read as 0 (the frame's first or last bytes)
__device__ __forceinline__ unsigned rec_bytes4(const unsigned char* p, const unsigned char* hi) {
  unsigned v = 0;
  for (int k = 0; k < 4 && p + k < hi; ++k) v |= (unsigned) p[k] << (8 * k);
  return v;
}
__device__ __forceinline__ unsigned rec_low_bytes(unsigned u, int len) { return len >= 4 ? u : (u & ((1u << (8 * len)) - 1u)); }

// the 4 bytes at p (any alignment) of the frame [lo, hi); bytes at or beyond hi read as 0 (p >= lo)
__device__ __forceinline__ unsigned rec_src4(const unsigned char* p, const unsigned char* lo, const unsigned char* hi) {
  const unsigned char* a = (const unsigned char*) ((uintptr_t) p & ~(uintptr_t) 3);
  const int sh = (int) ((uintptr_t) p & 3) * 8;
  if (a >= lo && a + (sh ? 8 : 4) <= hi) {
    const unsigned w0 = rec_ld4(a), w1 = sh ? rec_ld4(a + 4) : 0u;
    return (unsigned) ((((unsigned long long) w1 << 32) | w0) >> sh);
  }
  return rec_bytes4(p, hi);
}

// One tile of a record gather, run by every thread of the CTA: output record i (0 <= i < cnt <= rec_tile_pts(step)) = source
// record idx[i0 + i] of the frame [lo, hi), written to a + i * step. s_w and s_idx are the caller's shared arrays.
__device__ __forceinline__ void rec_gather_tile(const unsigned char* lo, const unsigned char* hi, int step, const int* __restrict__ idx, long long i0,
                                                int cnt, unsigned char* a, unsigned* s_w, int* s_idx) {
  const int tid = threadIdx.x;
  for (int i = tid; i < cnt; i += REC_THREADS) s_idx[i] = idx[i0 + i];
  unsigned char* b = a + (size_t) cnt * step;               // the tile's bytes [a, b) of dst
  unsigned char* a_floor = (unsigned char*) ((uintptr_t) a & ~(uintptr_t) 15);   // shared word 0 stands for this address
  const int r0 = (int) (a - a_floor), r1 = r0 + cnt * step;   // the tile's bytes in shared memory
  __syncthreads();
  // shared word w: tile bytes t = 4w + j - r0 (r0 <= 4w + j < r1), byte t % step of source record s_idx[t / step]
  const int w_beg = r0 >> 2, w_end = (r1 + 3) >> 2;
  if (step < 4) {
    // a word may hold bytes of up to four records: one piece per record it touches
    for (int w = w_beg + tid; w < w_end; w += REC_THREADS) {
      int j = r0 - 4 * w > 0 ? r0 - 4 * w : 0;
      const int je = r1 - 4 * w < 4 ? r1 - 4 * w : 4;
      const int t = 4 * w + j - r0;
      int i = t / step, c = t - i * step;
      unsigned v = 0;
      while (j < je) {
        const int len = je - j < step - c ? je - j : step - c;
        v |= rec_low_bytes(rec_src4(lo + (long long) s_idx[i] * step + c, lo, hi), len) << (8 * j);
        j += len;
        ++i;
        c = 0;
      }
      s_w[w] = v;
    }
  } else {
    // step >= 4: a word holds piece A (record i from its byte c) and, where records meet, piece B (record i + 1 from byte 0).
    // Pass 1 issues the two aligned loads of every piece of REC_GW words (predicated off where they would leave the frame);
    // pass 2 re-aligns and combines them, with byte loads for the pieces at the frame's two ends.
    for (int wb = w_beg + tid; wb < w_end; wb += REC_GW * REC_THREADS) {
      unsigned la0[REC_GW], la1[REC_GW], lb0[REC_GW], lb1[REC_GW];
      const unsigned char* pa[REC_GW];
      const unsigned char* pb[REC_GW];
      int ja[REC_GW], na[REC_GW], nb[REC_GW];
      bool oka[REC_GW], okb[REC_GW];
#pragma unroll
      for (int q = 0; q < REC_GW; ++q) {
        const int w = wb + q * REC_THREADS;
        int i = 0, c = 0, j0 = 0, je = 0;
        if (w < w_end) {
          j0 = r0 - 4 * w > 0 ? r0 - 4 * w : 0;
          je = r1 - 4 * w < 4 ? r1 - 4 * w : 4;
          const int t = 4 * w + j0 - r0;
          i = t / step;
          c = t - i * step;
        }
        ja[q] = j0;
        na[q] = je - j0 < step - c ? je - j0 : step - c;   // 0 past the tile
        nb[q] = je - j0 - na[q];
        pa[q] = lo + (long long) s_idx[i] * step + c;
        pb[q] = nb[q] > 0 ? lo + (long long) s_idx[i + 1] * step : lo;
        const unsigned char* a4 = (const unsigned char*) ((uintptr_t) pa[q] & ~(uintptr_t) 3);
        const unsigned char* b4 = (const unsigned char*) ((uintptr_t) pb[q] & ~(uintptr_t) 3);
        oka[q] = na[q] > 0 && a4 >= lo && a4 + 8 <= hi;
        okb[q] = nb[q] > 0 && b4 >= lo && b4 + 8 <= hi;
        la0[q] = oka[q] ? rec_ld4(a4) : 0u;
        la1[q] = oka[q] ? rec_ld4(a4 + 4) : 0u;
        lb0[q] = okb[q] ? rec_ld4(b4) : 0u;
        lb1[q] = okb[q] ? rec_ld4(b4 + 4) : 0u;
      }
#pragma unroll
      for (int q = 0; q < REC_GW; ++q) {
        const int w = wb + q * REC_THREADS;
        if (w >= w_end) continue;
        const int sa = (int) ((uintptr_t) pa[q] & 3) * 8, sb = (int) ((uintptr_t) pb[q] & 3) * 8;
        const unsigned ua = oka[q] ? (unsigned) ((((unsigned long long) la1[q] << 32) | la0[q]) >> sa) : rec_bytes4(pa[q], hi);
        unsigned v = rec_low_bytes(ua, na[q]) << (8 * ja[q]);
        if (nb[q] > 0) {
          const unsigned ub = okb[q] ? (unsigned) ((((unsigned long long) lb1[q] << 32) | lb0[q]) >> sb) : rec_bytes4(pb[q], hi);
          v |= rec_low_bytes(ub, nb[q]) << (8 * (ja[q] + na[q]));
        }
        s_w[w] = v;
      }
    }
  }
  __syncthreads();
  const unsigned char* s_b = reinterpret_cast<const unsigned char*>(s_w);
  unsigned char* a16 = (unsigned char*) (((uintptr_t) a + 15) & ~(uintptr_t) 15);
  unsigned char* b16 = (unsigned char*) ((uintptr_t) b & ~(uintptr_t) 15);
  if (a16 < b16) {
    const int nvec = (int) ((b16 - a16) >> 4), vbase = (int) (a16 - a_floor);
#pragma unroll 4
    for (int k = tid; k < nvec; k += REC_THREADS) rec_st16(a16 + 16 * k, s_b + vbase + 16 * k);
    const int head = (int) (a16 - a), tail = (int) (b - b16);
    if (tid < head) a[tid] = s_b[r0 + tid];
    else if (tid >= 16 && tid < 16 + tail) b16[tid - 16] = s_b[(b16 - a_floor) + (tid - 16)];
  } else {
    for (int k = tid; k < (int) (b - a); k += REC_THREADS) a[k] = s_b[r0 + k];
  }
}

// frame f = blockIdx.y: output records [k0, k0 + tile) of its region. recs / pt_off / rec_off / nd are the call's tables (the
// unpack's record table, point offsets, byte offsets of the output regions, dropped counts), idx the index lists.
__global__ void __launch_bounds__(REC_THREADS, 4) k_gather_records(const RecordFrame* __restrict__ recs, const long long* __restrict__ pt_off,
                                                                 const long long* __restrict__ rec_off, const int* __restrict__ nd,
                                                                 const int* __restrict__ idx,
                                                                 unsigned char* __restrict__ dst) {
  __shared__ __align__(16) unsigned s_w[REC_SMEM_WORDS];
  __shared__ int s_idx[REC_MAX_TILE_PTS];
  const int f = blockIdx.y;
  const long long p0 = pt_off[f];
  const long long n = pt_off[f + 1] - p0;
  const long long m = n - nd[f];                       // ground + non-ground records of the frame
  const int step = recs[f].step;
  const int tp = rec_tile_pts(step);
  const long long k0 = (long long) blockIdx.x * tp;
  if (k0 >= m) return;
  const int cnt = (int) (m - k0 < tp ? m - k0 : tp);
  const unsigned char* lo = recs[f].src;
  rec_gather_tile(lo, lo + n * step, step, idx, p0 + k0, cnt, dst + rec_off[f] + k0 * step, s_w, s_idx);
}

// ---- record results of a bound call (pwpp_bind_record_results): one buffer per part, regions fixed by the capacities -------
//
// k_gather_record_parts writes part z = first + blockIdx.z (0 ground, 1 non-ground) of frame f = blockIdx.y: output record k of
// the part's list = input record idx[start + k], to dst_z + part_off[f] + k * step. The list is found on the device: the ground
// list starts at pt_off[f] and holds counts[f] records, the non-ground list follows it and holds n - counts[f] - counts[2 nf + f]
// (counts: the call's count rows, num_ground, num_patches, num_dropped). The grid is sized from the capacities, so CTAs past the
// list return at once; CTA (0, f, 0) writes both counts of the frame to part_cnt[2f], part_cnt[2f + 1], whichever parts run.
// Frame f's tiles stay inside [part_off[f], part_off[f] + count * step) and read only [src, src + n * step).
//
// k_gather_record_packed (pwpp_bind_packed_records) is the same gather into packed records: every frame of the call has the
// same step, g_off / ng_off are each part's record offsets (k_bound_xyz_offsets, in records), and frame f's list of a part goes
// to dst_z + off_z[f] * step with no padding between frames, so neighbouring frames may share a 16-byte word (rec_gather_tile
// writes only its own bytes). It writes no counts. Frame f's tiles stay inside [off_z[f] * step, off_z[f + 1] * step).
template <bool Packed>
__device__ __forceinline__ void gather_record_parts_body(const RecordFrame* __restrict__ recs, const long long* __restrict__ pt_off,
                                                         const int* __restrict__ counts, int nf, const int* __restrict__ idx,
                                                         const long long* __restrict__ g_off, const long long* __restrict__ ng_off, int first,
                                                         unsigned char* __restrict__ ground, unsigned char* __restrict__ nonground,
                                                         int* __restrict__ part_cnt, unsigned* s_w, int* s_idx) {
  const int f = blockIdx.y, part = first + (int) blockIdx.z;
  const long long p0 = pt_off[f];
  const long long n = pt_off[f + 1] - p0;
  const int ng = counts[f];
  const long long nn = n - ng - counts[2 * nf + f];
  if (!Packed && blockIdx.x == 0 && blockIdx.z == 0 && threadIdx.x == 0) { part_cnt[2 * f] = ng; part_cnt[2 * f + 1] = (int) nn; }
  const long long m = part ? nn : ng;
  const int step = recs[f].step;
  const int tp = rec_tile_pts(step);
  const long long k0 = (long long) blockIdx.x * tp;
  if (k0 >= m) return;
  const int cnt = (int) (m - k0 < tp ? m - k0 : tp);
  const unsigned char* lo = recs[f].src;
  unsigned char* dst = part ? nonground : ground;
  const long long o = Packed ? (part ? ng_off : g_off)[f] * step : g_off[f];   // the byte offset of the frame's region
  rec_gather_tile(lo, lo + n * step, step, idx, p0 + (part ? ng : 0) + k0, cnt, dst + o + k0 * step, s_w, s_idx);
}

__global__ void __launch_bounds__(REC_THREADS, 4) k_gather_record_parts(const RecordFrame* __restrict__ recs, const long long* __restrict__ pt_off,
                                                                      const int* __restrict__ counts, int nf, const int* __restrict__ idx,
                                                                      const long long* __restrict__ part_off, int first,
                                                                      unsigned char* __restrict__ ground, unsigned char* __restrict__ nonground,
                                                                      int* __restrict__ part_cnt) {
  __shared__ __align__(16) unsigned s_w[REC_SMEM_WORDS];
  __shared__ int s_idx[REC_MAX_TILE_PTS];
  gather_record_parts_body<false>(recs, pt_off, counts, nf, idx, part_off, part_off, first, ground, nonground, part_cnt, s_w, s_idx);
}

__global__ void __launch_bounds__(REC_THREADS, 4) k_gather_record_packed(const RecordFrame* __restrict__ recs, const long long* __restrict__ pt_off,
                                                                       const int* __restrict__ counts, int nf, const int* __restrict__ idx,
                                                                       const long long* __restrict__ g_off, const long long* __restrict__ ng_off,
                                                                       int first, unsigned char* __restrict__ ground,
                                                                       unsigned char* __restrict__ nonground) {
  __shared__ __align__(16) unsigned s_w[REC_SMEM_WORDS];
  __shared__ int s_idx[REC_MAX_TILE_PTS];
  gather_record_parts_body<true>(recs, pt_off, counts, nf, idx, g_off, ng_off, first, ground, nonground, nullptr, s_w, s_idx);
}

// Byte offsets of every frame's output region (16-byte aligned, room for all n[f] records): off[nf + 1].
inline void rec_out_offsets(const long long* pt_off, const RecordFrame* recs, int nf, long long* off) {
  off[0] = 0;
  for (int f = 0; f < nf; ++f) off[f + 1] = off[f] + (((pt_off[f + 1] - pt_off[f]) * recs[f].step + 15) & ~15LL);
}

// grid.x of k_gather_record_parts over frames of these capacities: the tiles of the largest, at least 1 (the counts are written)
inline long long rec_parts_grid_x(const long long* cap_off, const RecordFrame* recs, int nf) {
  const long long gx = rec_grid_x(cap_off, recs, nf);
  return gx > 0 ? gx : 1;
}

}  // namespace pwpp

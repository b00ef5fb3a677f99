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

// frame f = blockIdx.y: output records [k0, k0 + tile) of its region. recs / pt_off / rec_off / nd are the call's tables (the
// unpack's record table, point offsets, byte offsets of the output regions, dropped counts), idx the index lists.
__global__ void __launch_bounds__(REC_THREADS, 4) k_gather_records(const RecordFrame* __restrict__ recs, const long long* __restrict__ pt_off,
                                                                 const long long* __restrict__ rec_off, const int* __restrict__ nd,
                                                                 const int* __restrict__ idx,
                                                                 unsigned char* __restrict__ dst) {
  __shared__ __align__(16) unsigned s_w[REC_SMEM_WORDS];
  __shared__ int s_idx[REC_MAX_TILE_PTS];
  const int f = blockIdx.y, tid = threadIdx.x;
  const long long p0 = pt_off[f];
  const long long n = pt_off[f + 1] - p0;
  const long long m = n - nd[f];                       // ground + non-ground records of the frame
  const int step = recs[f].step;
  const int tp = rec_tile_pts(step);
  const long long k0 = (long long) blockIdx.x * tp;
  if (k0 >= m) return;
  const int cnt = (int) (m - k0 < tp ? m - k0 : tp);
  const unsigned char* lo = recs[f].src;
  const unsigned char* hi = lo + n * step;
  for (int i = tid; i < cnt; i += REC_THREADS) s_idx[i] = idx[p0 + k0 + i];
  unsigned char* a = dst + rec_off[f] + k0 * step;          // the tile's bytes [a, b) of dst
  unsigned char* b = a + (size_t) cnt * step;
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

// Byte offsets of every frame's output region (16-byte aligned, room for all n[f] records): off[nf + 1].
inline void rec_out_offsets(const long long* pt_off, const RecordFrame* recs, int nf, long long* off) {
  off[0] = 0;
  for (int f = 0; f < nf; ++f) off[f + 1] = off[f] + (((pt_off[f + 1] - pt_off[f]) * recs[f].step + 15) & ~15LL);
}

}  // namespace pwpp

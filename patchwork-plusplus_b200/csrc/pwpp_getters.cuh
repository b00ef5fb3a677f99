// pwpp_getters.cuh — the reference's getters of a bound call on the device (pwpp_bind_getter_results, include/pwpp.h):
// getGround / getNonground as float32 xyz rows and getHeight's state, written into fixed buffers at every run or replay.
//
// k_gather_xyz_parts is the bound call's k_gather_xyz: one launch over every frame and both parts, grid sized from the
// capacities, each list found on the device (as k_gather_record_parts finds it). k_gather_xyz_packed is the same gather into
// packed rows (pwpp_bind_packed_xyz), whose per-frame starts k_bound_xyz_offsets scans on the device first. k_gather_record_parts cannot serve here: its
// tile copies whole records of one step, and an xyz row is a 12-byte prefix of the ctx's 16-byte point. The rows are read
// from the ctx's float4 input, the cloud the direct call's xyz getters read, so a row is bit for bit what they return.
// k_bound_states converts, after each run, the state of every frame's stream into a pwpp_state row.
#pragma once
#include "pwpp_common.cuh"
#include "pwpp_gle.cuh"
#include "pwpp_records.cuh"
#include "pwpp.h"

namespace pwpp {

constexpr int XYZ_THREADS = 256;
constexpr int XYZ_PER_THREAD = 4;   // points a thread has in flight: index loads, then point loads, then stores
constexpr int XYZ_TILE = XYZ_THREADS * XYZ_PER_THREAD;

// Part z = first + blockIdx.z (0 ground, 1 non-ground) of frame f = blockIdx.y: row k of the part = xyz of point
// idx[start + k] of the frame, written to dst_z + 3 (row_off_z[f] + k). The ground list starts at pt_off[f] and holds counts[f]
// points; the non-ground list follows it and holds n - counts[f] - counts[2 nf + f] (counts: the call's count rows num_ground,
// num_patches, num_dropped). CTAs past the list return at once. No row past a count is written.
// k_gather_xyz_parts (the capacity layout: one row_off for both parts) also has CTA (0, f, 0) write both counts of the frame to
// xyz_cnt[2f], xyz_cnt[2f + 1], whichever parts run; k_gather_xyz_packed takes one row-offset array per part (k_bound_xyz_offsets).
template <bool Packed>
__device__ __forceinline__ void gather_xyz_body(const float4* __restrict__ pts, const long long* __restrict__ pt_off, const int* __restrict__ counts,
                                                int nf, const int* __restrict__ idx, const long long* __restrict__ g_off,
                                                const long long* __restrict__ ng_off, int first, float* __restrict__ ground,
                                                float* __restrict__ nonground, int* __restrict__ xyz_cnt) {
  const int f = blockIdx.y, part = first + (int) blockIdx.z;
  const long long p0 = pt_off[f];
  const long long n = pt_off[f + 1] - p0;
  const int ng = counts[f];
  const long long nn = n - ng - counts[2 * nf + f];
  if (!Packed && blockIdx.x == 0 && blockIdx.z == 0 && threadIdx.x == 0) { xyz_cnt[2 * f] = ng; xyz_cnt[2 * f + 1] = (int) nn; }
  const long long m = part ? nn : ng;
  const long long k0 = (long long) blockIdx.x * XYZ_TILE;
  if (k0 >= m) return;
  const int cnt = (int) (m - k0 < XYZ_TILE ? m - k0 : XYZ_TILE);
  const int* li = idx + p0 + (part ? ng : 0) + k0;
  const float4* src = pts + p0;
  float* out = (part ? nonground : ground) + (((Packed && part) ? ng_off : g_off)[f] + k0) * 3;
  int j[XYZ_PER_THREAD];
  float4 v[XYZ_PER_THREAD];
#pragma unroll
  for (int u = 0; u < XYZ_PER_THREAD; ++u) {
    const int i = (int) threadIdx.x + u * XYZ_THREADS;
    j[u] = i < cnt ? __ldg(li + i) : 0;
  }
#pragma unroll
  for (int u = 0; u < XYZ_PER_THREAD; ++u) {
    const int i = (int) threadIdx.x + u * XYZ_THREADS;
    if (i < cnt) v[u] = __ldg(src + j[u]);
  }
#pragma unroll
  for (int u = 0; u < XYZ_PER_THREAD; ++u) {
    const int i = (int) threadIdx.x + u * XYZ_THREADS;
    if (i < cnt) { out[3 * i] = v[u].x; out[3 * i + 1] = v[u].y; out[3 * i + 2] = v[u].z; }
  }
}

__global__ void __launch_bounds__(XYZ_THREADS) k_gather_xyz_parts(const float4* __restrict__ pts, const long long* __restrict__ pt_off,
                                                                  const int* __restrict__ counts, int nf, const int* __restrict__ idx,
                                                                  const long long* __restrict__ row_off, int first, float* __restrict__ ground,
                                                                  float* __restrict__ nonground, int* __restrict__ xyz_cnt) {
  gather_xyz_body<false>(pts, pt_off, counts, nf, idx, row_off, row_off, first, ground, nonground, xyz_cnt);
}

__global__ void __launch_bounds__(XYZ_THREADS) k_gather_xyz_packed(const float4* __restrict__ pts, const long long* __restrict__ pt_off,
                                                                   const int* __restrict__ counts, int nf, const int* __restrict__ idx,
                                                                   const long long* __restrict__ g_off, const long long* __restrict__ ng_off,
                                                                   int first, float* __restrict__ ground, float* __restrict__ nonground) {
  gather_xyz_body<true>(pts, pt_off, counts, nf, idx, g_off, ng_off, first, ground, nonground, nullptr);
}

// k_bound_xyz_offsets: one CTA after the last run of a bound call with packed xyz (pwpp_bind_packed_xyz). g_off and ng_off
// (nf + 1 entries each) receive the exclusive scans of every frame's ground count counts[f] and non-ground list length
// n - counts[f] - counts[2 nf + f], so frame f's packed rows of a part start at its entry and the totals end each array.
// Thread t owns a contiguous slice of frames, as in bound_table_body, and the slices are scanned the same way.
__global__ void __launch_bounds__(BT_THREADS) k_bound_xyz_offsets(int nf, const long long* __restrict__ pt_off, const int* __restrict__ counts,
                                                                  long long* __restrict__ g_off, long long* __restrict__ ng_off) {
  __shared__ long long s_g[BT_THREADS / 32];
  __shared__ long long s_n[BT_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (nf + BT_THREADS - 1) / BT_THREADS;
  const int f0 = tid * per < nf ? tid * per : nf;
  const int f1 = f0 + per < nf ? f0 + per : nf;
  long long own_g = 0, own_n = 0;
  for (int f = f0; f < f1; ++f) {
    own_g += counts[f];
    own_n += pt_off[f + 1] - pt_off[f] - counts[f] - counts[2 * nf + f];
  }
  long long g, nn;   // the start of the slice
  bt_scan_slices(lane, warp, own_g, own_n, g, nn, s_g, s_n);
  for (int f = f0; f < f1; ++f) {
    g_off[f] = g;
    ng_off[f] = nn;
    g += counts[f];
    nn += pt_off[f + 1] - pt_off[f] - counts[f] - counts[2 * nf + f];
  }
  if (tid == BT_THREADS - 1) { g_off[nf] = g; ng_off[nf] = nn; }   // the last slice ends at the totals
}

// grid.x of k_gather_xyz_parts over frames of these capacities (cap_off: their prefix sum): the tiles of the largest, at least 1
// (the counts are written)
inline long long xyz_parts_grid_x(const long long* cap_off, int nf) {
  long long gx = 1;
  for (int f = 0; f < nf; ++f) {
    const long long t = (cap_off[f + 1] - cap_off[f] + XYZ_TILE - 1) / XYZ_TILE;
    gx = t > gx ? t : gx;
  }
  return gx;
}

// Frames [f0, f1) of one run, after its k_gle: out[f] = the state of frame f's stream b_stream[f], the bound stream table. A
// skipped frame's own entry in the run's stream table names its scratch slot; the bound table names the real stream, which
// no other frame of the run writes (a run's streams are pairwise distinct), so it reads the state as the stream's earlier
// frames left it.
constexpr int BS_THREADS = 128;

__device__ __forceinline__ void bound_state_row(const StreamState& s, pwpp_state* __restrict__ out) {
  pwpp_state r;
  r.sensor_height = s.sensor_height;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r.elevation_thr[i] = s.elevation_thr[i];
    r.flatness_thr[i] = s.flatness_thr[i];
    r.n_elevation[i] = s.n_elev[i];
    r.n_flatness[i] = s.n_flat[i];
  }
  *out = r;
}

__global__ void __launch_bounds__(BS_THREADS) k_bound_states(int f0, int f1, const int* __restrict__ b_stream, const StreamState* __restrict__ states,
                                                             pwpp_state* __restrict__ out) {
  const int f = f0 + (int) (blockIdx.x * BS_THREADS + threadIdx.x);
  if (f >= f1) return;
  bound_state_row(states[b_stream[f]], out + f);
}

// The same with a stream table (pwpp_bind_stream_table): the stream is the one frame f read (the run's copy, read). A frame
// skipped by its action or as a duplicate still names a stream: its row is that stream's state after the run (a duplicate's
// stream was run by the frame that won it). A hole or an out-of-range id leaves its row as it was.
__global__ void __launch_bounds__(BS_THREADS) k_bound_states_streams(int f0, int f1, const int* __restrict__ read, int num_streams,
                                                                     const StreamState* __restrict__ states, pwpp_state* __restrict__ out) {
  const int f = f0 + (int) (blockIdx.x * BS_THREADS + threadIdx.x);
  if (f >= f1) return;
  const int s = read[f];
  if (s >= 0 && s < num_streams) bound_state_row(states[s], out + f);
}

}  // namespace pwpp

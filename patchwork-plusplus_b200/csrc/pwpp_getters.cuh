// pwpp_getters.cuh — the reference's getters of a bound call on the device (pwpp_bind_getter_results, include/pwpp.h):
// getGround / getNonground as float32 xyz rows and getHeight's state, written into fixed buffers at every run or replay.
//
// k_gather_xyz_parts is the bound call's k_gather_xyz: one launch over every frame and both parts, grid sized from the
// capacities, each list found on the device (as k_gather_record_parts finds it). k_gather_record_parts cannot serve here: its
// tile copies whole records of one step, and an xyz row is a 12-byte prefix of the ctx's 16-byte point. The rows are read
// from the ctx's float4 input, the cloud the direct call's xyz getters read, so a row is bit for bit what they return.
// k_bound_states converts, after each run, the state of every frame's stream into a pwpp_state row.
#pragma once
#include "pwpp_common.cuh"
#include "pwpp_gle.cuh"
#include "pwpp.h"

namespace pwpp {

constexpr int XYZ_THREADS = 256;
constexpr int XYZ_PER_THREAD = 4;   // points a thread has in flight: index loads, then point loads, then stores
constexpr int XYZ_TILE = XYZ_THREADS * XYZ_PER_THREAD;

// Part z = first + blockIdx.z (0 ground, 1 non-ground) of frame f = blockIdx.y: row k of the part = xyz of point
// idx[start + k] of the frame, written to dst_z + 3 (row_off[f] + k). The ground list starts at pt_off[f] and holds counts[f]
// points; the non-ground list follows it and holds n - counts[f] - counts[2 nf + f] (counts: the call's count rows num_ground,
// num_patches, num_dropped). CTAs past the list return at once; CTA (0, f, 0) writes both counts of the frame to
// xyz_cnt[2f], xyz_cnt[2f + 1], whichever parts run. No row past a count is written.
__global__ void __launch_bounds__(XYZ_THREADS) k_gather_xyz_parts(const float4* __restrict__ pts, const long long* __restrict__ pt_off,
                                                                  const int* __restrict__ counts, int nf, const int* __restrict__ idx,
                                                                  const long long* __restrict__ row_off, int first, float* __restrict__ ground,
                                                                  float* __restrict__ nonground, int* __restrict__ xyz_cnt) {
  const int f = blockIdx.y, part = first + (int) blockIdx.z;
  const long long p0 = pt_off[f];
  const long long n = pt_off[f + 1] - p0;
  const int ng = counts[f];
  const long long nn = n - ng - counts[2 * nf + f];
  if (blockIdx.x == 0 && blockIdx.z == 0 && threadIdx.x == 0) { xyz_cnt[2 * f] = ng; xyz_cnt[2 * f + 1] = (int) nn; }
  const long long m = part ? nn : ng;
  const long long k0 = (long long) blockIdx.x * XYZ_TILE;
  if (k0 >= m) return;
  const int cnt = (int) (m - k0 < XYZ_TILE ? m - k0 : XYZ_TILE);
  const int* li = idx + p0 + (part ? ng : 0) + k0;
  const float4* src = pts + p0;
  float* out = (part ? nonground : ground) + (row_off[f] + k0) * 3;
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

__global__ void __launch_bounds__(BS_THREADS) k_bound_states(int f0, int f1, const int* __restrict__ b_stream, const StreamState* __restrict__ states,
                                                             pwpp_state* __restrict__ out) {
  const int f = f0 + (int) (blockIdx.x * BS_THREADS + threadIdx.x);
  if (f >= f1) return;
  const StreamState& s = states[b_stream[f]];
  pwpp_state r;
  r.sensor_height = s.sensor_height;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r.elevation_thr[i] = s.elevation_thr[i];
    r.flatness_thr[i] = s.flatness_thr[i];
    r.n_elevation[i] = s.n_elev[i];
    r.n_flatness[i] = s.n_flat[i];
  }
  out[f] = r;
}

}  // namespace pwpp

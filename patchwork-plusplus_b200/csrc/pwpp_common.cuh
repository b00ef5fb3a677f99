// pwpp_common.cuh — small device helpers and launch geometry shared by all kernels.
#pragma once
#include <cuda_runtime.h>

#include "pwpp_gle.cuh"
#include "pwpp_math.cuh"

namespace pwpp {

constexpr int CHUNK_PTS = 4096;      // points per CTA in k_bin_hist / k_scatter
constexpr int CHUNK_THREADS = 256;   // 8 warps, each owns 512 consecutive points
constexpr int WARP_PTS = CHUNK_PTS / (CHUNK_THREADS / 32);  // 512
constexpr int WARP_ITERS = WARP_PTS / 32;                   // 16
constexpr int MAX_LPR = 64;          // num_lpr supported by the warp selection buffer
constexpr int MAX_RVPF = 8;          // num_iter supported (R-VPF planes kept in registers)

#if defined(PWPP_SIMT_EMU)
// tests/simt (the kernels run on the CPU): the stream table of a FrameTable whose initializer names none. It is the identity
// table (frame f -> stream f, what the twin's multi-frame calls mean) unless a harness points it at another table for the
// duration of a call. Device builds have no default: pwpp_capi.cu always passes the call's table.
inline const int* simt_identity_streams() {
  static int v[65536];
  static const bool filled = [] { for (int i = 0; i < 65536; ++i) v[i] = i; return true; }();
  (void) filled;
  return v;
}
inline const int* g_simt_streams = simt_identity_streams();
// the parameter-set table of a FrameTable whose initializer names none: every frame on set 0 (a one-set context), unless a
// harness points it at another table for the duration of a call
inline const int* simt_zero_sets() {
  static int v[65536] = {};
  return v;
}
inline const int* g_simt_sets = simt_zero_sets();
#ifndef __grid_constant__
#define __grid_constant__
#endif
#endif

struct FrameTable {            // per call, device arrays indexed by frame
  const long long* pt_off;     // [F+1] first point of each frame in the packed point array
  const int* chunk_off;        // [F+1] first chunk of each frame
  // [F] stream of each frame: index of its StreamState and of its history rows
#if defined(PWPP_SIMT_EMU)
  const int* stream = g_simt_streams;
  const int* pset = g_simt_sets;
#else
  const int* stream;
  const int* pset;             // [F] parameter set of each frame (the set of its stream): index into GeometrySets / AlgoParamSets
#endif
};

// The parameter sets of a context (pwpp_create_sets), passed BY VALUE to every kernel that reads them: the records sit in the
// kernel's parameter bank, and a kernel reads its frame's record through a reference into it (`__grid_constant__`: no local
// copy), one indexed constant load per field. Not a __constant__ symbol (contexts on one device would share it), not a global
// table (the fit kernels have no registers to spare for the extra pointer and loads). A one-set context fills set 0 only; the
// converting constructors make a single Geometry / AlgoParams the set table of a one-set launch.
constexpr int MAX_PARAM_SETS = 8;   // PWPP_MAX_PARAM_SETS
struct GeometrySets {
  Geometry g[MAX_PARAM_SETS];
  int nbs;                     // stride of the per-frame bin arrays (patch records, centers, normals): the largest nbins of the sets
  GeometrySets() = default;
  __host__ __device__ GeometrySets(const Geometry& g0) : g{g0}, nbs(g0.nbins) {}
};
struct AlgoParamSets {
  AlgoParams a[MAX_PARAM_SETS];
  AlgoParamSets() = default;
  __host__ __device__ AlgoParamSets(const AlgoParams& a0) : a{a0} {}
};
// both tables plus the other arguments of the kernel with the longest list (k_front_cluster: < 256 bytes) stay inside the
// classic 4 KB kernel-parameter limit
static_assert(sizeof(GeometrySets) + sizeof(AlgoParamSets) + 256 <= 4096, "parameter-set tables exceed the kernel parameter space");
// history row capacity of a set (DESIGN.md section 3, deviation 1): the newest hcap samples of a ring are kept
__host__ __device__ inline int history_cap(const Geometry& g, const AlgoParams& ap) {
  int ms = 0;
  for (int k = 0; k < 4; ++k) ms = g.num_sectors[k] > ms ? g.num_sectors[k] : ms;
  return (ap.max_elevation_storage > ap.max_flatness_storage ? ap.max_elevation_storage : ap.max_flatness_storage) + 4 * ms + 64;
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
// ---- thread-block clusters (k_front_cluster): rank, barrier, distributed shared memory ----
#if defined(PWPP_SIMT_EMU)
__device__ __forceinline__ unsigned pw_cluster_rank() { return blockIdx.x; }                 // the twin launches one cluster at a time, blockIdx.x = rank
__device__ __forceinline__ void pw_cluster_sync() { simt::cluster_sync_(); }
template <typename T> __device__ __forceinline__ T* pw_cluster_map(T* p, unsigned rank) { return static_cast<T*>(simt::cluster_map_(p, (int) rank)); }
#else
}  // namespace pwpp
#include <cooperative_groups.h>
namespace pwpp {
__device__ __forceinline__ unsigned pw_cluster_rank() { return cooperative_groups::this_cluster().block_rank(); }
__device__ __forceinline__ void pw_cluster_sync() { cooperative_groups::this_cluster().sync(); }
template <typename T> __device__ __forceinline__ T* pw_cluster_map(T* p, unsigned rank) { return cooperative_groups::this_cluster().map_shared_rank(p, rank); }
#endif

#if defined(PWPP_SIMT_EMU)   // tests/simt: the kernels compiled by g++ and run lane by lane on the CPU (test infrastructure only)
__device__ __forceinline__ unsigned lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) { return *p; }
__device__ __forceinline__ void prefetch_l2(const void*) {}
#else
// dynamic shared memory of a kernel, typed (tests/simt/cuda_runtime.h defines the CPU counterpart)
#define PW_DYN_SHARED(T, name) extern __shared__ T name[]
__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  // read-once data: bypass L1 allocation, keep L2 normal
  float4 v;
  asm("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#endif

// ---- bulk async copy global -> shared::cta (the TMA engine; a contiguous range needs no tensor map; SASS: UBLKCP), completion
// on an mbarrier ----
#if !defined(PWPP_SIMT_EMU)
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif


}  // namespace pwpp

// pwpp_capi.cu — implementation of the C-ABI declared in include/pwpp.h (libpwpp_b200.so).
// Host side only orchestrates: every stage of estimateGround() runs in the kernels of pwpp_kernels.cuh.
// There is no CPU fallback; without a CUDA device pwpp_create() fails with PWPP_ERR_NO_DEVICE.
#include <cuda_runtime.h>

#include <sched.h>

#include <algorithm>
#include <cctype>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "pwpp.h"
#include "pwpp_kernels.cuh"
#include "pwpp_records.cuh"
#include "pwpp_getters.cuh"
#include "pwpp_state_copy.cuh"
#include "pwpp_ladder.cuh"
#include "pwpp_tuning.h"
#include "pwpp_host.hpp"

using namespace pwpp;

static_assert(sizeof(BinFit) == sizeof(pwpp_bin_result), "BinFit must mirror pwpp_bin_result");
static_assert(sizeof(pwpp_scan_ring) == 32, "pwpp_scan_ring is a 32-byte record");
static_assert(sizeof(pwpp_state) == 104, "pwpp_state is a 104-byte record");

namespace {

thread_local std::string g_last_error;

// integer experiment switch from the environment, clamped to [lo, hi]
int env_int(const char* name, int dflt, int lo, int hi) {
  const char* e = std::getenv(name);
  if (!e || !*e) return dflt;
  const long v = std::strtol(e, nullptr, 10);
  return (int) (v < lo ? lo : (v > hi ? hi : v));
}

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define CU_TRY(expr)                                                                                         \
  do {                                                                                                       \
    cudaError_t _e = (expr);                                                                                 \
    if (_e != cudaSuccess) {                                                                                 \
      return fail(PWPP_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
    }                                                                                                        \
  } while (0)

unsigned long long g_alloc_gen = 0;   // bumped whenever a device buffer moves: captured CUDA graphs hold the old pointers

// InGraphs = false: a buffer no captured launch sequence reads (its moves leave the graphs valid).
// A buffer owns its allocation: it frees it when destroyed, and a move hands it over and leaves the source empty.
template <typename T, bool InGraphs = true>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); o.release(); return *this; }
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (InGraphs) ++g_alloc_gen;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 8 + 64;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // reserve that keeps the contents (synchronous); when the allocation fails the buffer stays as it was
  cudaError_t grow_keep(size_t n) {
    if (n <= cap) return cudaSuccess;
    const size_t want = n + n / 8 + 64;
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p) e = cudaMemcpy(q, p, cap * sizeof(T), cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) { cudaFree(q); return e; }
    if (InGraphs) ++g_alloc_gen;
    if (p) cudaFree(p);
    p = q;
    cap = want;
    return cudaSuccess;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  PinBuf(PinBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  PinBuf& operator=(PinBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); o.release(); return *this; }
  ~PinBuf() { release(); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 8 + 64;
    cudaError_t e = cudaMallocHost(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

}  // namespace

// N x cols column-major (an Eigen::MatrixXf, reference patchworkpp.h:152) -> packed float4 {x, y, z, intensity | 0}
__global__ void k_repack_colmajor(const float* __restrict__ src, long long n, int cols, float4* __restrict__ dst) {
  const long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = make_float4(src[i], src[n + i], src[2 * n + i], cols == 4 ? src[3 * n + i] : 0.f);
}

// packed N x 3 rows on the device (the ROS node's conversion, reference ros/src/Utils.hpp:158-172) -> float4 {x, y, z, 0}
__global__ void k_pad_xyz(const float* __restrict__ src, long long n, float4* __restrict__ dst) {
  const long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = make_float4(src[3 * i], src[3 * i + 1], src[3 * i + 2], 0.f);
}

typedef void (*FitKernel)(const float4*, FrameTable, const StreamState*, GeometrySets, AlgoParamSets, int, const int*, WorkQueues, int*, BinFit*);
struct FitLaunch {
  FitKernel fn = nullptr;
  int grid = 0, threads = 0;
  size_t smem = 0;
};
typedef void (*Ref32Kernel)(const float4*, FrameTable, const StreamState*, GeometrySets, AlgoParamSets, const int*, WorkQueues, int*, BinFit*, Ref32Scratch, int);
struct Ref32Launch {
  Ref32Kernel fn = nullptr;
  int grid = 0, threads = 0;
  size_t smem = 0;
};

constexpr int NUM_SIDE = 6;

// A bound call's width ladder (pwpp_bind_width_ladder): the selector's widths, one plain graph per width holding the call's launch
// sequence cut at that width (enqueue_bound_body), and the whole run (table, selector, SWITCH node) as an executable graph for
// runs on a stream that is not capturing.
struct BoundLadder {
  LadderWidths widths{};
  std::vector<cudaGraph_t> bodies;
  cudaGraphExec_t exec = nullptr;
  long long body_launches = 0;   // launches of the widest body: the same call's count without a ladder, less the table kernel
  long long launches = 0;        // launches of one run
  BoundLadder() = default;
  BoundLadder(const BoundLadder&) = delete;
  BoundLadder& operator=(const BoundLadder&) = delete;
  ~BoundLadder() {
    if (exec) cudaGraphExecDestroy(exec);
    for (cudaGraph_t g : bodies) cudaGraphDestroy(g);
  }
};

struct pwpp_ctx {
  // parameter sets (pwpp_create: one) and the set of every stream; the kernels get the set records by value
  int num_sets = 1;
  std::vector<pwpp_params> set_params;      // the sets as created (pwpp_clone)
  GeometrySets gs;                          // gs.nbs: the largest bin count of the sets, stride of the per-frame bin arrays
  AlgoParamSets aps;
  bool set_fast[MAX_PARAM_SETS] = {};       // build_geometry: the fp32 binning filter is exact for the set's geometry
  int set_hcap[MAX_PARAM_SETS] = {};        // history row capacity of the set (history_cap)
  std::vector<int> stream_set;              // [num_streams]
  int device = 0;
  int num_streams = 0;
  int nbp = 0;          // padded number of bins incl. pseudo-bins, of the set with the most bins
  int hist_stride = 0;  // row stride of d_hist in doubles: the largest set_hcap
  // kernel-variant switches, read from the environment when the context is created (see pwpp_create)
  int sw_front = 1, sw_patch = 0, small_call_frames = 0;
  bool sw_serial_fit = false, front_dense_ok = false;
  cudaStream_t stream = nullptr, stream_h2d = nullptr, stream_d2h = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_begin = nullptr, ev_end = nullptr;
  bool call_times_valid = false;
  cudaEvent_t stage_ev[PWPP_NUM_STAGES + 1] = {};
  cudaStream_t side[NUM_SIDE] = {};       // one side stream per patch-size class: its fit kernel, then its sort (reference order)
  cudaEvent_t ev_fork = nullptr, ev_fit[NUM_SIDE] = {}, ev_join[NUM_SIDE] = {};
  bool profiling = false, stage_valid = false;
  long long launches = 0;

  // persistent per-stream state
  DevBuf<StreamState> d_states;
  DevBuf<StreamState> d_states_init;  // constructor state of every stream (reset source)
  DevBuf<double> d_hist;
  DevBuf<int> d_stream_hcap;          // [num_streams] history capacity of every stream's set (device state copies)
  DevBuf<int> d_claim;                // [num_streams] claim table of pwpp_import_states_device, -1 between calls

  // per-call work buffers
  DevBuf<float4> d_in;            // host path only
  DevBuf<float> d_cm;             // host path: column-major frames as uploaded, repacked on the device
  DevBuf<long long> d_pt_off;     // [F+1]
  DevBuf<int> d_chunk_off;        // [F+1]
  DevBuf<int> d_stream;           // [F] stream of every frame of the call
  DevBuf<int> d_pset;             // [F] parameter set of every frame of the call
  DevBuf<unsigned short> d_bin_ids;
  DevBuf<unsigned short> d_chist;
  DevBuf<unsigned int> d_cbase;
  DevBuf<int> d_bin_off;          // [F][nbp+1]
  DevBuf<float4> d_sorted;
  DevBuf<int> d_part;
  DevBuf<BinFit> d_fits;          // [F][nbins]
  DevBuf<BinSeg> d_segs;          // [F][nbins+3]
  DevBuf<int4> d_wq_items[NUM_CLASSES];  // fit work queues
  DevBuf<int> d_wq_ctr;           // [2*NUM_CLASSES + 2*ORD_NUM_HEADS]: counts, heads, the heads of the five k_order and five k_order_exact launches
  DevBuf<unsigned char> d_labels; // reference-order output only: what became of every point of a fitted patch
  DevBuf<unsigned> d_ox_scratch;  // PWPP_ORDER_REFERENCE_EXACT only: workspace of the fix-up above 512 points, OX_X_WORDS words per point
  DevBuf<unsigned long long> d_ox_counts;   // [OX_NUM_STATS] counters of the fix-up (pwpp_order_exact_counts)
  int order_mode = 0;             // PWPP_ORDER_*
  int arith = PWPP_ARITH_DOUBLE;  // PWPP_ARITH_*: the fit kernels and the k_gle instantiation of launch_range_impl
  Ref32Launch fit_ref32[NUM_CLASSES];   // k_fit_ref32 of every patch-size class (PWPP_ARITH_REFERENCE)
  // PWPP_ARITH_REFERENCE only: storage of the patches above the shared capacity of their k_fit_ref32 (Ref32Scratch)
  DevBuf<unsigned long long> d_r32_keys;
  DevBuf<float4> d_r32_pts;
  DevBuf<float> d_r32_sel;
  DevBuf<unsigned char> d_r32_flags;
  FitLaunch fit[NUM_CLASSES];   // persistent fit kernel of every patch-size class (variant chosen in pwpp_create)
  FitLaunch fit_small[NUM_CLASSES];   // the same for calls of at most small_call_frames frames (one CTA per patch above 512 points)
  int max_sectors = 0;
  FitLaunch order_k[ORD_NUM_HEADS];   // k_order_cta<512, X>, <512, L3>, <256, L2>, <128, L1>, k_order_warp (same argument list as the fit kernels' type is not needed: launched by name)
  FitLaunch exact_k[ORD_NUM_HEADS];   // k_order_exact_big<X>, <L3>, <L2>, <L1>, k_order_exact_warp: grid, threads and shared memory of each
  DevBuf<int> d_out_idx;
  DevBuf<int> d_counts;           // [3][F]: num_ground, num_patches, num_dropped (F = frames of the call)
  DevBuf<float> d_centers, d_normals;  // [F][nbins][3]
  DevBuf<float> d_xyz;            // gather scratch
  DevBuf<unsigned char> d_raw;    // pwpp_estimate_host_records: the frames' records as uploaded, unpacked on the device
  DevBuf<RecordFrame> d_rec;      // [F] record table of a records call
  // record results (pwpp_*_record_results), reserved by the first call that asks for them
  DevBuf<unsigned char, false> d_rec_out;   // every frame's ground and non-ground records, region f at rec_off[f]
  DevBuf<long long, false> d_rec_off;       // [F+1]

  PinBuf<float4> h_in;
  PinBuf<long long> h_pt_off_buf[2];      // double-buffered: a call never waits for the previous call's upload
  PinBuf<int> h_chunk_off_buf[2];
  PinBuf<int> h_stream_buf[2];
  PinBuf<int> h_pset_buf[2];
  PinBuf<RecordFrame> h_rec_buf[2];
  PinBuf<unsigned char> h_raw;            // page-locked staging of pageable records
  PinBuf<long long> h_rec_off;            // upload of rec_off; ev_rec_off marks when the copy has read it
  PinBuf<unsigned char> h_rec_out;        // host view of d_rec_out
  cudaEvent_t ev_rec_off = nullptr;
  cudaEvent_t tab_ev[2] = {nullptr, nullptr};
  int tab_cur = 0;
  std::vector<int> chunk_off;             // host copy of the current call's chunk table
  std::vector<int> frame_set;             // host copy of the current call's set table
  // Frames of one stream are sequentially dependent (k_gle of one frame writes what the next one reads), so a call is
  // launched as runs of consecutive frames with pairwise distinct streams: frames [runs[r], runs[r + 1]) are run r.
  std::vector<int> runs;
  std::vector<int> identity;              // [num_streams] 0, 1, 2, ...: the stream table of pwpp_estimate_host / _device
  std::vector<int> last_pos;              // [num_streams] scratch of the run split, -1 between calls
  PinBuf<int> h_out_idx;
  PinBuf<int> h_counts;
  PinBuf<float> h_centers, h_normals;

  // description of the last call
  int last_nframes = 0;
  long long last_total = 0;
  std::vector<long long> pt_off;  // host copy
  const float4* last_pts = nullptr;  // device pointer of the input of the last call
  bool counts_fetched = false, idx_fetched = false, patches_fetched = false;
  std::vector<RecordFrame> last_recs;     // record table of the last call when it took records (empty otherwise)
  std::vector<long long> rec_off;         // [F+1] byte offsets of the record result regions (set by the gather)
  bool rec_gathered = false, rec_fetched = false;
  double last_time_us = 0.0;
  cudaStream_t last_stream = nullptr;
  int last_call = -1;             // the bound call that is the last call (make_bound_last), -1: a direct call
  bool off_fetched = false;       // the last call's point offsets were fetched (fetch_offsets)

  // a bound call (pwpp_bind_call): what its runs re-establish and launch, and the device buffers it owns (released with it).
  // The work buffers are frozen while any call is bound.
  struct Bound {
    bool on = false;
    int nf = 0, has_intensity = 0;
    const long long* d_counts = nullptr;    // the caller's device counts
    std::vector<int> runs, frame_set, cap_chunk_off;
    std::vector<long long> cap_pt_off;      // the capacity layout: sizes grids and picks the dense front end only
    DevBuf<long long, false> d_bmax;        // [F] max_n
    DevBuf<int, false> d_bstream, d_bpset;  // [F] the bound call's stream and set tables
    DevBuf<int, false> d_bstatus;           // [F] PWPP_COUNT_OUT_OF_RANGE or 0
    std::vector<RecordFrame> recs;          // its record table (host copy of d_brec)
    DevBuf<RecordFrame, false> d_brec;      // [F] its record table
    int rec_parts = 0;                      // record results (pwpp_bind_record_results): PWPP_PART_* bits, 0 = off
    std::vector<long long> rec_part_off;    // [F+1] byte offsets of every frame's region in each part buffer
    DevBuf<unsigned char, false> d_bground, d_bnonground;   // its record results, one buffer per part (region f at rec_part_off[f])
    DevBuf<long long, false> d_bpart_off;   // [F+1] rec_part_off
    DevBuf<int, false> d_rec_counts;        // [F][2]: ground, non-ground records of every frame of the last run
    const int* d_actions = nullptr;         // the caller's device actions (pwpp_bind_call_actions), NULL: none
    std::vector<char> reset_run;            // [runs] the run holds a frame whose stream ran in an earlier run: k_bound_reset
    DevBuf<int, false> d_bscratch, d_bdep;  // [F] with actions: scratch slot of every frame; its stream has a frame in an earlier run
    DevBuf<int, false> d_bact;              // [F] the run's copy of the actions
    const int* d_slots = nullptr;           // the caller's device slots (pwpp_bind_call_rings), NULL: no rings
    DevBuf<BoundRing, false> d_bring;       // [F] with rings: every frame's ring
    DevBuf<int, false> d_bslot;             // [F] the run's copy of the slots
    DevBuf<RecordFrame, false> d_brun;      // [F] the run's record table (d_brec with every frame's slot or offset applied)
    const long long* d_offsets = nullptr;   // the caller's device offsets (pwpp_bind_call_packed), NULL: not packed
    long long capacity = 0;                 // records at the packed buffer's base
    int getters = 0;                        // getter results (pwpp_bind_getter_results): PWPP_GETTER_* bits, 0 = off
    DevBuf<float, false> d_bgxyz, d_bngxyz;  // getter results: [sum(max_n)][3] ground / non-ground xyz, frame f from row cap_pt_off[f]
    DevBuf<long long, false> d_bxyz_off;    // [F+1] cap_pt_off
    DevBuf<int, false> d_xyz_counts;        // [F][2]: ground, non-ground xyz rows of every frame of the last run
    DevBuf<pwpp_state, false> d_bstates;    // [F] the state of every frame's stream right after the frame
    int packed_xyz = 0;                     // packed xyz results (pwpp_bind_packed_xyz): PWPP_PART_* bits, 0 = off
    DevBuf<float, false> d_pgxyz, d_pngxyz;  // [sum(max_n)][3] packed ground / non-ground xyz
    DevBuf<long long, false> d_pg_off, d_png_off;   // [F+1] ground / non-ground offsets of packed xyz and packed records, scanned
                                                     // on the device at every run when either is enabled
    int packed_rec = 0;                     // packed records (pwpp_bind_packed_records): PWPP_PART_* bits, 0 = off
    DevBuf<unsigned char, false> d_prec_g, d_prec_ng;   // [sum(max_n)][point_step] packed ground / non-ground records
    const int* d_streams = nullptr;         // the caller's device streams (pwpp_bind_stream_table), NULL: the bound stream table
    DevBuf<int, false> d_bread;             // [F] with a stream table: the run's copy of the streams
    DevBuf<int, false> d_bclaim;            // [num_streams] its duplicate claims, -1 between runs
    DevBuf<int, false> d_bset_of;           // [num_streams] stream_set, for the sets of the streams read on the device
    DevBuf<int, false> d_bruns;             // [runs + 1] runs, for the duplicate check run by run
    bool ran = false;                       // a run was enqueued or captured: the state buffers may no longer move
    DevBuf<int, false> d_width;             // the width the last run launched (pwpp_bound_call_width)
    std::unique_ptr<BoundLadder> ladder;    // its width ladder (pwpp_bind_width_ladder), NULL: none
  };
  // Bound calls 0 .. PWPP_MAX_BOUND_CALLS - 1. They share the stream states, the scratch slots and the work buffers, so a bind
  // may grow those only while none of them has run (check_growth).
  Bound bound[PWPP_MAX_BOUND_CALLS];
  int sel = 0;                            // the call the bind, run, result and unbind entry points act on (pwpp_select_bound_call)
  int scratch_slots = 0;                  // state / history slots after the streams' (the longest run of any bind), kept after unbind
  bool sets_on_device = false;            // the last call's sets were picked on the device (a stream table): range_fast asks every
                                          // set, and fetch_offsets fetches frame_set

  // small calls (the reference's one-frame-per-call pattern): the launch sequence replayed as a CUDA graph
  struct GraphKey { int nf, call_frames, has_intensity, chunks, fast, arith; unsigned long long gen; const void* pts; };
  cudaGraphExec_t gexec[2] = {nullptr, nullptr};
  GraphKey gkey[2] = {};
  long long glaunches[2] = {0, 0};
  int sw_graph = 1;

  // frees every buffer (pwpp_destroy); not exported: the context is opaque to callers
  __attribute__((visibility("hidden"))) ~pwpp_ctx() = default;
};

namespace {

int validate_params(const pwpp_params* p) {
  if (!p) return fail(PWPP_ERR_INVALID_ARG, "params is NULL");
  if (p->num_zones != PWPP_NUM_ZONES) return fail(PWPP_ERR_UNSUPPORTED, "num_zones must be 4 (the reference hard-wires four zones, patchworkpp.h:127-134)");
  if (p->num_rings_of_interest < 0 || p->num_rings_of_interest > PWPP_MAX_RINGS_OF_INTEREST)
    return fail(PWPP_ERR_UNSUPPORTED, "num_rings_of_interest must be in [0,4] (patchworkpp.h:174-175 holds 4 histories)");
  if (p->num_min_pts < 0) return fail(PWPP_ERR_UNSUPPORTED, "num_min_pts must be >= 0");
  if (p->num_iter < 1 || p->num_iter > MAX_RVPF) return fail(PWPP_ERR_UNSUPPORTED, "num_iter must be in [1,8]");
  if (p->num_lpr < 1 || p->num_lpr > MAX_LPR) return fail(PWPP_ERR_UNSUPPORTED, "num_lpr must be in [1,64]");
  if (!(p->th_seeds > 0) || !(p->th_seeds_v > 0)) return fail(PWPP_ERR_UNSUPPORTED, "th_seeds and th_seeds_v must be > 0");
  if (!(p->max_range > p->min_range) || !(p->min_range >= 0)) return fail(PWPP_ERR_INVALID_ARG, "need 0 <= min_range < max_range");
  if (p->max_flatness_storage < 1 || p->max_elevation_storage < 1) return fail(PWPP_ERR_INVALID_ARG, "max_*_storage must be >= 1");
  long long nb = 0;
  for (int k = 0; k < 4; ++k) {
    if (p->num_rings_each_zone[k] < 1 || p->num_sectors_each_zone[k] < 1 || p->num_sectors_each_zone[k] > 1024)
      return fail(PWPP_ERR_UNSUPPORTED, "rings per zone must be >= 1 and sectors per zone in [1,1024]");
    nb += (long long) p->num_rings_each_zone[k] * p->num_sectors_each_zone[k];
  }
  if (nb + PW_NUM_PSEUDO > 4096) return fail(PWPP_ERR_UNSUPPORTED, "more than 4093 bins are not supported");
  return PWPP_OK;
}

// The dynamic shared-memory limit is an attribute of the kernel, shared by every context of the process: a context only ever
// raises it, so that a context whose geometry needs less (fewer bins, fewer sectors) does not break the launches of one that
// needs more.
template <typename F>
cudaError_t raise_smem_limit(F* fn, size_t bytes) {
  cudaFuncAttributes a;
  const cudaError_t e = cudaFuncGetAttributes(&a, (const void*) fn);
  if (e != cudaSuccess) return e;
  if ((size_t) a.maxDynamicSharedSizeBytes >= bytes) return cudaSuccess;
  return cudaFuncSetAttribute((const void*) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bytes);
}

int bind_device(pwpp_ctx* ctx) {
  CU_TRY(cudaSetDevice(ctx->device));
  return PWPP_OK;
}

// Checks the stream table of a call: 1 <= nframes <= 65535 (a grid dimension of the per-frame kernels), every id a stream of
// the ctx. Nothing is launched and no state changes when it fails.
int check_streams(const pwpp_ctx* ctx, int nframes, const int32_t* streams) {
  if (!streams) return fail(PWPP_ERR_INVALID_ARG, "streams is NULL");
  if (nframes < 1 || nframes > 65535) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, 65535]");
  for (int f = 0; f < nframes; ++f)
    if (streams[f] < 0 || streams[f] >= ctx->num_streams)
      return fail(PWPP_ERR_INVALID_ARG, "stream id " + std::to_string(streams[f]) + " of frame " + std::to_string(f) + " is outside [0, num_streams)");
  return PWPP_OK;
}

// Splits a call into maximal runs of consecutive frames whose streams are pairwise distinct (ctx->runs).
void split_runs(pwpp_ctx* ctx, int nframes, const int32_t* streams) {
  ctx->runs.assign(1, 0);
  for (int f = 0; f < nframes; ++f) {
    int& p = ctx->last_pos[streams[f]];
    if (p >= ctx->runs.back()) ctx->runs.push_back(f);   // the stream already has a frame in the current run
    p = f;
  }
  ctx->runs.push_back(nframes);
  for (int f = 0; f < nframes; ++f) ctx->last_pos[streams[f]] = -1;
}

// The work buffers of a call over nframes frames, total points and total_chunks chunks (and the input buffer, with_input).
// With check_only nothing is allocated: PWPP_ERR_CAPACITY when one of them would have to grow (frozen by a bound call).
int reserve_work(pwpp_ctx* ctx, int nframes, long long total, long long total_chunks, bool with_input, bool check_only) {
  const size_t nb = ctx->gs.nbs, nbp = ctx->nbp, nb_all = nb + PW_NUM_PSEUDO, nf = (size_t) nframes, np = (size_t) total;
  bool grow = false;
  cudaError_t err = cudaSuccess;
  auto need = [&](auto& b, size_t n) {
    if (check_only) grow = grow || n > b.cap;
    else if (err == cudaSuccess) err = b.reserve(n);
  };
  if (with_input) need(ctx->d_in, std::max<size_t>(np, 1));
  need(ctx->d_pt_off, nf + 1);
  need(ctx->d_chunk_off, nf + 1);
  need(ctx->d_stream, nf);
  need(ctx->d_pset, nf);
  need(ctx->d_bin_ids, np);
  need(ctx->d_chist, (size_t) total_chunks * nbp);
  need(ctx->d_cbase, (size_t) total_chunks * nbp);
  need(ctx->d_bin_off, nf * (nbp + 1));
  need(ctx->d_sorted, np);
  need(ctx->d_part, np);
  if (ctx->order_mode) need(ctx->d_labels, np);
  if (ctx->order_mode == PWPP_ORDER_REFERENCE_EXACT) need(ctx->d_ox_scratch, (size_t) OX_X_WORDS * std::max<size_t>(np, 1));
  if (ctx->arith == PWPP_ARITH_REFERENCE) {
    need(ctx->d_r32_keys, 2 * std::max<size_t>(np, 1));
    need(ctx->d_r32_pts, std::max<size_t>(np, 1));
    need(ctx->d_r32_sel, 3 * std::max<size_t>(np, 1));
    need(ctx->d_r32_flags, 2 * std::max<size_t>(np, 1));
  }
  need(ctx->d_fits, nf * nb);
  need(ctx->d_segs, nf * nb_all);
  for (int c = 0; c < NUM_CLASSES; ++c) need(ctx->d_wq_items[c], nf * nb);
  need(ctx->d_out_idx, np);
  need(ctx->d_counts, 3 * nf);
  need(ctx->d_centers, nf * nb * 3);
  need(ctx->d_normals, nf * nb * 3);
  if (grow)
    return fail(PWPP_ERR_CAPACITY, "a call of " + std::to_string(nframes) + " frames and " + std::to_string(total) +
                                       " points does not fit the work buffers frozen by the bound calls (unbinding every bound call lifts the freeze)");
  if (err != cudaSuccess) return fail(PWPP_ERR_CUDA, std::string("reserving the work buffers: ") + cudaGetErrorString(err));
  return PWPP_OK;
}

bool any_bound(const pwpp_ctx* ctx) {
  for (const pwpp_ctx::Bound& b : ctx->bound)
    if (b.on) return true;
  return false;
}

// A bind (nframes > 0: frames, total points, chunks) or a stream-table enable (nframes = 0) that needs slots scratch slots, while
// another bound call has run or been captured: its graphs hold the work and state buffers, so neither may move.
// PWPP_ERR_CAPACITY, before anything changes, when either would have to grow. With no run yet everything grows as needed.
int check_growth(pwpp_ctx* ctx, int slots, int nframes = 0, long long total = 0, long long chunks = 0) {
  bool ran = false;
  for (const pwpp_ctx::Bound& b : ctx->bound) ran = ran || b.ran;
  if (!ran) return PWPP_OK;
  const std::string fix = ", and another bound call has run or been captured: bind every call, widest first, before the first run or capture";
  if (slots > ctx->scratch_slots)
    return fail(PWPP_ERR_CAPACITY, "the call needs " + std::to_string(slots) + " scratch state slots (its longest run), the ctx has " +
                                       std::to_string(ctx->scratch_slots) + fix);
  if (nframes > 0 && reserve_work(ctx, nframes, total, chunks, true, true))
    return fail(PWPP_ERR_CAPACITY, "a call of " + std::to_string(nframes) + " frames and " + std::to_string(total) +
                                       " points (the sum of max_n) needs larger work buffers" + fix);
  return PWPP_OK;
}

// A direct call while a call is bound: PWPP_ERR_CAPACITY, before anything runs or changes, when the call would grow a work
// buffer. Frame f has n[f] points (negative sizes were refused by the caller).
int check_frozen(pwpp_ctx* ctx, int nframes, const int64_t* n, bool with_input) {
  if (!any_bound(ctx)) return PWPP_OK;
  long long total = 0, chunks = 0;
  for (int f = 0; f < nframes; ++f) {
    total += n[f];
    chunks += (n[f] + CHUNK_PTS - 1) / CHUNK_PTS;
  }
  return reserve_work(ctx, nframes, total, chunks, with_input, true);
}

// Sizes the work buffers for a call over nframes frames (ctx->pt_off filled), uploads the frame tables (points, chunks,
// stream of every frame and, for a records call, the record table) and splits the call into runs.
int prepare_call(pwpp_ctx* ctx, int nframes, const int32_t* streams, cudaStream_t s, const RecordFrame* recs = nullptr) {
  const long long total = ctx->pt_off[nframes];
  int total_chunks = 0;
  ctx->tab_cur ^= 1;
  const int tb = ctx->tab_cur;
  PinBuf<long long>& h_pt_off = ctx->h_pt_off_buf[tb];
  PinBuf<int>& h_chunk_off = ctx->h_chunk_off_buf[tb];
  PinBuf<int>& h_stream = ctx->h_stream_buf[tb];
  PinBuf<int>& h_pset = ctx->h_pset_buf[tb];
  CU_TRY(cudaEventSynchronize(ctx->tab_ev[tb]));   // upload issued two calls ago: long finished
  CU_TRY(h_pt_off.reserve(nframes + 1));
  CU_TRY(h_chunk_off.reserve(nframes + 1));
  CU_TRY(h_stream.reserve(nframes));
  CU_TRY(h_pset.reserve(nframes));
  std::memcpy(h_stream.p, streams, (size_t) nframes * sizeof(int));
  ctx->frame_set.resize(nframes);
  for (int f = 0; f < nframes; ++f) h_pset.p[f] = ctx->frame_set[f] = ctx->stream_set[streams[f]];
  split_runs(ctx, nframes, streams);
  ctx->chunk_off.assign(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const long long n = ctx->pt_off[f + 1] - ctx->pt_off[f];
    if (n < 0 || n > 0x7fffffffLL - CHUNK_PTS) return fail(PWPP_ERR_INVALID_ARG, "frame size out of range");
    h_pt_off.p[f] = ctx->pt_off[f];
    h_chunk_off.p[f] = total_chunks;
    ctx->chunk_off[f] = total_chunks;
    total_chunks += (int) ((n + CHUNK_PTS - 1) / CHUNK_PTS);
  }
  h_pt_off.p[nframes] = total;
  h_chunk_off.p[nframes] = total_chunks;
  ctx->chunk_off[nframes] = total_chunks;
  const int rc = reserve_work(ctx, nframes, total, total_chunks, false, false);
  if (rc) return rc;
  CU_TRY(cudaMemcpyAsync(ctx->d_pt_off.p, h_pt_off.p, (nframes + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ctx->d_chunk_off.p, h_chunk_off.p, (nframes + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ctx->d_stream.p, h_stream.p, nframes * sizeof(int), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ctx->d_pset.p, h_pset.p, nframes * sizeof(int), cudaMemcpyHostToDevice, s));
  if (recs) ctx->last_recs.assign(recs, recs + nframes);
  else ctx->last_recs.clear();
  ctx->rec_gathered = ctx->rec_fetched = false;
  if (recs) {
    PinBuf<RecordFrame>& h_rec = ctx->h_rec_buf[tb];
    CU_TRY(h_rec.reserve(nframes));
    CU_TRY(ctx->d_rec.reserve(nframes));
    std::memcpy(h_rec.p, recs, (size_t) nframes * sizeof(RecordFrame));
    CU_TRY(cudaMemcpyAsync(ctx->d_rec.p, h_rec.p, nframes * sizeof(RecordFrame), cudaMemcpyHostToDevice, s));
  }
  CU_TRY(cudaEventRecord(ctx->tab_ev[tb], s));
  ctx->last_nframes = nframes;
  ctx->last_total = total;
  ctx->last_call = -1;
  ctx->sets_on_device = false;
  ctx->counts_fetched = ctx->idx_fetched = ctx->patches_fetched = false;
  ctx->stage_valid = false;
  return PWPP_OK;
}

// The fp32 binning filter is used for a launch range only when build_geometry allows it for every set the range names;
// otherwise the range takes the exact kernel. Both bin exactly, so the bins are the same either way. When the sets are picked on
// the device (a bound stream table) the host does not know them: every set of the ctx must allow it.
bool range_fast(const pwpp_ctx* ctx, int f0, int nf) {
  if (ctx->sets_on_device) {
    for (int k = 0; k < ctx->num_sets; ++k)
      if (!ctx->set_fast[k]) return false;
    return true;
  }
  for (int f = f0; f < f0 + nf; ++f)
    if (!ctx->set_fast[ctx->frame_set[f]]) return false;
  return true;
}

// Launches the whole path for frames [f0, f0 + nf) of the prepared call on stream s; the range must not hold two frames of
// one stream (a run or part of one). A frame range is the same launch sequence over per-frame arrays offset by f0 (frame
// tables hold absolute point / chunk positions), which is what lets pwpp_estimate_host pipeline chunks of frames against
// their H2D / D2H copies. Stream state and histories are indexed by the stream table, never by the frame.
// The kernel variants (small-call kernels, dense front end, fp32 binning filter) are those of frames [vf0, vf0 + vnf), by default
// the range itself: a width-ladder body launches parts of a run with the run's variants, whose results it must reproduce.
int launch_range_impl(pwpp_ctx* ctx, int f0, int nf, const float4* d_pts, int has_intensity, cudaStream_t s, bool prof, int chunks_override,
                      int vf0 = -1, int vnf = 0) {
  if (vnf <= 0) { vf0 = f0; vnf = nf; }
  int max_chunks = 0;
  for (int f = f0; f < f0 + nf; ++f) max_chunks = std::max(max_chunks, ctx->chunk_off[f + 1] - ctx->chunk_off[f]);
  if (chunks_override > 0) max_chunks = chunks_override;   // graph capture: grids sized for a range of frame sizes (surplus CTAs exit at once)
  if (chunks_override < 0) max_chunks = 0;                 // frames the bound table kernel rejected: empty on every run
  const int nb = ctx->gs.nbs, nbp = ctx->nbp, nb_all = nb + PW_NUM_PSEUDO;   // strides of the per-frame bin arrays (the largest set)
  const int nframes = nf;
  FrameTable ft{ctx->d_pt_off.p + f0, ctx->d_chunk_off.p + f0, ctx->d_stream.p + f0, ctx->d_pset.p + f0};
  const bool fast = range_fast(ctx, vf0, vnf);
  StreamState* states = ctx->d_states.p;
  double* hist = ctx->d_hist.p;
  int* bin_off = ctx->d_bin_off.p + (size_t) f0 * (nbp + 1);
  BinFit* fits = ctx->d_fits.p + (size_t) f0 * nb;
  BinSeg* segs = ctx->d_segs.p + (size_t) f0 * nb_all;
  float* centers = ctx->d_centers.p + (size_t) f0 * nb * 3;
  float* normals = ctx->d_normals.p + (size_t) f0 * nb * 3;
  CU_TRY(cudaMemsetAsync(ctx->d_wq_ctr.p, 0, (2 * NUM_CLASSES + 2 * ORD_NUM_HEADS) * sizeof(int), s));
  int stage = 0;
#define STAGE_MARK() do { if (prof) CU_TRY(cudaEventRecord(ctx->stage_ev[stage], s)); ++stage; } while (0)
  STAGE_MARK();
  WorkQueues wq;
  for (int c = 0; c < NUM_CLASSES; ++c) wq.items[c] = ctx->d_wq_items[c].p;
  wq.count = ctx->d_wq_ctr.p;
  wq.head = ctx->d_wq_ctr.p + NUM_CLASSES;
  wq.labels = ctx->order_mode ? ctx->d_labels.p : nullptr;
  // A call of a few frames (the reference's pattern is one frame per call) cannot fill the GPU with warp-sized work items: there the
  // latency of the longest patch counts, so patches above 512 points go to the CTA-per-patch kernels, and one frame's cloud is
  // binned by ~30 independent CTAs (the three stand-alone kernels) rather than by the 8 CTAs of one cluster: both shorten
  // the longest kernel of a one-frame call.
  const bool small_call = vnf <= ctx->small_call_frames;
  const FitLaunch* fitk = small_call ? ctx->fit_small : ctx->fit;
  if (ctx->sw_front && !small_call) {
    // one thread-block cluster per frame: binning, scan and stable scatter in one kernel (pwpp_front.cuh)
    if (nframes > 0) {
      // 64 warps per frame for KITTI-sized frames, 128 for dense ones (pwpp_front.cuh)
      const long long mean_front = (ctx->pt_off[vf0 + vnf] - ctx->pt_off[vf0]) / std::max(vnf, 1);
      const bool dense = mean_front > 400000 && ctx->front_dense_ok;
      const int nt = dense ? FC_THREADS_DENSE : FC_THREADS;
      const size_t sm_f = front_cluster_smem_bytes(nbp, nt);
      dim3 grid(FC_CS, nframes);
#define FC_ARGS d_pts, ft, states, ctx->gs, ctx->aps, has_intensity, nbp, nb, ctx->d_bin_ids.p, bin_off, wq, fits, ctx->d_sorted.p
      if (dense) {
        if (fast) k_front_cluster<true, CLS_L2_MAX, FC_THREADS_DENSE><<<grid, nt, sm_f, s>>>(FC_ARGS);
        else k_front_cluster<false, CLS_L2_MAX, FC_THREADS_DENSE><<<grid, nt, sm_f, s>>>(FC_ARGS);
      } else {
        if (fast) k_front_cluster<true, CLS_L2_MAX, FC_THREADS><<<grid, nt, sm_f, s>>>(FC_ARGS);
        else k_front_cluster<false, CLS_L2_MAX, FC_THREADS><<<grid, nt, sm_f, s>>>(FC_ARGS);
      }
#undef FC_ARGS
      ++ctx->launches;
    }
    STAGE_MARK(); STAGE_MARK(); STAGE_MARK();
  } else {
    // the three stand-alone kernels (PWPP_FRONT=0)
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_h = nbp * sizeof(unsigned int);
#define HIST_ARGS d_pts, ft, states, ctx->gs, ctx->aps, has_intensity, nbp, ctx->d_bin_ids.p, ctx->d_chist.p
      if (!fast) k_bin_hist<false, 0><<<grid, CHUNK_THREADS, sm_h, s>>>(HIST_ARGS);
      else k_bin_hist<true, 2><<<grid, CHUNK_THREADS, sm_h, s>>>(HIST_ARGS);
#undef HIST_ARGS
      ++ctx->launches;
    }
    STAGE_MARK();
    k_bin_scan<CLS_L2_MAX><<<nframes, 512, (nbp + 1) * sizeof(int), s>>>(ft, nbp, nb, ctx->gs, ctx->aps, ctx->d_chist.p, ctx->d_cbase.p, bin_off, wq, fits);
    ++ctx->launches;
    STAGE_MARK();
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_sc = (size_t) (CHUNK_THREADS / 32) * nbp * sizeof(unsigned int);
      k_scatter<false, 4><<<grid, CHUNK_THREADS, sm_sc, s>>>(d_pts, ft, nbp, ctx->d_bin_ids.p, ctx->d_cbase.p, ctx->d_sorted.p);
      ++ctx->launches;
    }
    STAGE_MARK();
  }
  // persistent fit kernels, one per patch-size class (queues were filled by k_bin_scan). The classes are independent:
  // unless per-stage timing is requested they run on side streams so that the tail of one class (few long patches
  // left) overlaps the start of the next.
#define FIT_ARGS ctx->d_sorted.p, ft, states, ctx->gs, ctx->aps, nbp, bin_off, wq, ctx->d_part.p, fits
  const bool serial_fit = ctx->sw_serial_fit;   // PWPP_SERIAL_FIT: diagnostic switch
  // persistent grids are sized for a full GPU; a small call (one frame per call is the reference's pattern) would launch hundreds
  // of CTAs per class that find their queue empty and, worse, keep the six classes from running side by side: cap the grid
  // by what the call can hold (a frame has at most a few hundred patches)
  auto launch_fit = [&](int c, cudaStream_t st) {
    if (ctx->arith == PWPP_ARITH_REFERENCE) {   // the reference's fp32 fits (pwpp_fit_ref32.cuh), the same grid rule
      const Ref32Launch& k = ctx->fit_ref32[c];
      const Ref32Scratch scr{ctx->d_r32_keys.p, ctx->d_r32_pts.p, ctx->d_r32_sel.p, ctx->d_r32_flags.p};
      const long long cap = (long long) nframes * (k.threads <= 128 ? 96 : 48);
      const int grid = (int) std::min<long long>(k.grid, std::max<long long>(1, cap));
      k.fn<<<grid, k.threads, k.smem, st>>>(ctx->d_sorted.p, ft, states, ctx->gs, ctx->aps, bin_off, wq, ctx->d_part.p, fits, scr,
                                            ctx->order_mode == PWPP_ORDER_REFERENCE_EXACT ? 1 : 0);
      ++ctx->launches;
      return;
    }
    const FitLaunch& k = fitk[c];
    if (!k.fn) return;
    const long long cap = (long long) nframes * (k.threads <= 128 ? 96 : 48);
    const int grid = (int) std::min<long long>(k.grid, std::max<long long>(1, cap));
    k.fn<<<grid, k.threads, k.smem, st>>>(FIT_ARGS);
    ++ctx->launches;
  };
  // reference emission order inside every fitted patch (pwpp_order.cuh): one launch per class (X, L3, L2, L1 with a CTA sized to the
  // class; M + S one warp per patch). A sort only permutes `part` inside the patches of its own class, so it runs on its class's
  // side stream right behind the fit kernel, beside the other classes' fits and beside k_gle (which only reads the patch records);
  // k_emit joins everything. On a one-frame call the sort of the largest patch and the ring walk of k_gle are
  // both pure latency.
  int* heads = ctx->d_wq_ctr.p + 2 * NUM_CLASSES;
  auto launch_order = [&](int q, cudaStream_t so) {   // q: 0 = X, 1 = L3, 2 = L2, 3 = L1, 4 = M + S
    const int grid = (int) std::min<long long>(ctx->order_k[q].grid, std::max<long long>(1, (long long) nframes * (q == 4 ? 64 : 32)));
    const int th = ctx->order_k[q].threads;
    const size_t sm = ctx->order_k[q].smem;
    switch (q) {
      case 0: k_order_cta<512, 5><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      case 1: k_order_cta<512, 4><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      case 2: k_order_cta<256, 3><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      case 3: k_order_cta<128, 2><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      default: k_order_warp<<<grid, th, 0, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
    }
    ++ctx->launches;
    if (ctx->order_mode != PWPP_ORDER_REFERENCE_EXACT) return;
    // the libstdc++ order of equal z (pwpp_order_exact.cuh): behind the class's sort, on the same stream, its own ticket counter
    const int gx = (int) std::min<long long>(ctx->exact_k[q].grid, std::max<long long>(1, (long long) nframes * (q == 4 ? 64 : 32)));
    const int tx = ctx->exact_k[q].threads;
    const size_t smx = ctx->exact_k[q].smem;
    int* hx = heads + ORD_NUM_HEADS + q;
    unsigned* xws = ctx->d_ox_scratch.p;
    unsigned long long* cnt = ctx->d_ox_counts.p;
    switch (q) {
      case 0: k_order_exact_big<5><<<gx, tx, smx, so>>>(ctx->d_sorted.p, wq, hx, ctx->d_part.p, xws, cnt); break;
      case 1: k_order_exact_big<4><<<gx, tx, smx, so>>>(ctx->d_sorted.p, wq, hx, ctx->d_part.p, xws, cnt); break;
      case 2: k_order_exact_big<3><<<gx, tx, smx, so>>>(ctx->d_sorted.p, wq, hx, ctx->d_part.p, xws, cnt); break;
      case 3: k_order_exact_big<2><<<gx, tx, smx, so>>>(ctx->d_sorted.p, wq, hx, ctx->d_part.p, xws, cnt); break;
      default: k_order_exact_warp<<<gx, tx, smx, so>>>(ctx->d_sorted.p, wq, hx, ctx->d_part.p, cnt); break;
    }
    ++ctx->launches;
  };
  const bool aside = !(prof || serial_fit);
  if (!aside) {
    static const int order[NUM_CLASSES] = {0, 4, 3, 2, 1, 5};   // stage slots: S, L3, L2, L1, M, X
    for (int q = 0; q < NUM_CLASSES; ++q) { launch_fit(order[q], s); STAGE_MARK(); }
    if (ctx->order_mode) for (int q = 0; q < ORD_NUM_HEADS; ++q) launch_order(q, s);
  } else {
    // side stream of every class, longest patches first: L3, L2, L1, M, S, X
    static const int cls_of_side[NUM_SIDE] = {4, 3, 2, 1, 0, 5};
    static const int order_of_side[NUM_SIDE] = {1, 2, 3, 4, -1, 0};   // the sort that follows the fit on that stream (M + S: behind M)
    CU_TRY(cudaEventRecord(ctx->ev_fork, s));
    for (int q = 0; q < NUM_SIDE; ++q) {
      CU_TRY(cudaStreamWaitEvent(ctx->side[q], ctx->ev_fork, 0));
      launch_fit(cls_of_side[q], ctx->side[q]);
      CU_TRY(cudaEventRecord(ctx->ev_fit[q], ctx->side[q]));
    }
    if (ctx->order_mode) {
      for (int q = 0; q < NUM_SIDE; ++q) {
        if (order_of_side[q] < 0) continue;
        if (order_of_side[q] == 4) CU_TRY(cudaStreamWaitEvent(ctx->side[q], ctx->ev_fit[4], 0));   // the warp sort also covers class S (side 4)
        launch_order(order_of_side[q], ctx->side[q]);
        CU_TRY(cudaEventRecord(ctx->ev_join[q], ctx->side[q]));
      }
    }
    for (int q = 0; q < NUM_SIDE; ++q) CU_TRY(cudaStreamWaitEvent(s, ctx->ev_fit[q], 0));   // k_gle needs every fit, no sort
    stage += 6;
  }
#undef FIT_ARGS
  const int call_frames = ctx->last_nframes;   // the count rows are as long as the call
  int* d_ng = ctx->d_counts.p + f0;
  int* d_np = ctx->d_counts.p + call_frames + f0;
  int* d_nd = ctx->d_counts.p + 2 * call_frames + f0;
  {
    const size_t gle_smem = gle_smem_bytes(ctx->max_sectors);
    if (ctx->arith == PWPP_ARITH_REFERENCE)
      k_gle<true><<<nframes, 32, gle_smem, s>>>(ft, states, hist, ctx->hist_stride, ctx->gs, ctx->aps, nbp, ctx->max_sectors, bin_off, fits, segs, d_ng, d_np, centers, normals, d_nd);
    else
      k_gle<false><<<nframes, 32, gle_smem, s>>>(ft, states, hist, ctx->hist_stride, ctx->gs, ctx->aps, nbp, ctx->max_sectors, bin_off, fits, segs, d_ng, d_np, centers, normals, d_nd);
    ++ctx->launches;
  }
  STAGE_MARK();
  if (aside && ctx->order_mode) for (int q = 0; q < NUM_SIDE; ++q) if (q != 4) CU_TRY(cudaStreamWaitEvent(s, ctx->ev_join[q], 0));
  if (max_chunks > 0) {
    const long long max_pts = (long long) max_chunks * CHUNK_PTS;   // upper bound of the largest frame of the range
    dim3 grid((unsigned) ((max_pts + (long long) EMIT_TILE * EMIT_WARPS - 1) / ((long long) EMIT_TILE * EMIT_WARPS)), nframes);
    k_emit<<<grid, EMIT_WARPS * 32, 0, s>>>(ft, ctx->gs, nbp, bin_off, fits, segs, ctx->d_part.p, ctx->d_sorted.p, ctx->d_out_idx.p);
    ++ctx->launches;
  }
  STAGE_MARK();
#undef STAGE_MARK
  if (prof) ctx->stage_valid = true;
  CU_TRY(cudaGetLastError());
  ctx->last_pts = d_pts;
  ctx->last_stream = s;
  return PWPP_OK;
}

// Small calls are launch-bound (ten kernels of a few microseconds each plus the fork / join events of the fit kernels): the
// sequence is captured once per (frames, frames of the call, intensity flag, grid size class, binning kernel, buffer generation)
// and replayed as one CUDA graph; it reads the frame tables (stream and set ids included) the current call uploaded. Only for the
// first range of calls whose input sits in the ctx's own upload buffer (the host entry point), so the captured pointers
// stay valid; PWPP_GRAPH=0 switches it off.
constexpr int GRAPH_MAX_FRAMES = 16;
int launch_range(pwpp_ctx* ctx, int f0, int nf, const float4* d_pts, int has_intensity, cudaStream_t s, bool prof) {
  if (prof || !ctx->sw_graph || nf > GRAPH_MAX_FRAMES || f0 != 0 || d_pts != ctx->d_in.p) return launch_range_impl(ctx, f0, nf, d_pts, has_intensity, s, prof, 0);
  int max_chunks = 0;
  for (int f = 0; f < nf; ++f) max_chunks = std::max(max_chunks, ctx->chunk_off[f + 1] - ctx->chunk_off[f]);
  const int capc = std::max(8, (max_chunks + 7) & ~7);
  const int slot = has_intensity ? 1 : 0;
  const pwpp_ctx::GraphKey key{nf, ctx->last_nframes, has_intensity, capc, range_fast(ctx, 0, nf) ? 1 : 0, ctx->arith, g_alloc_gen, (const void*) d_pts};
  pwpp_ctx::GraphKey& have = ctx->gkey[slot];
  if (!ctx->gexec[slot] || have.nf != key.nf || have.call_frames != key.call_frames || have.chunks != key.chunks || have.fast != key.fast || have.arith != key.arith || have.gen != key.gen ||
      have.pts != key.pts) {
    if (ctx->gexec[slot]) { cudaGraphExecDestroy(ctx->gexec[slot]); ctx->gexec[slot] = nullptr; }
    const long long l0 = ctx->launches;
    CU_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int rc = launch_range_impl(ctx, 0, nf, d_pts, has_intensity, s, false, capc);
    cudaGraph_t graph = nullptr;
    const cudaError_t e = cudaStreamEndCapture(s, &graph);
    if (rc != PWPP_OK || e != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      ctx->sw_graph = 0;   // capture is not available here: fall back to plain launches for good
      ctx->launches = l0;
      return launch_range_impl(ctx, 0, nf, d_pts, has_intensity, s, false, 0);
    }
    const cudaError_t e2 = cudaGraphInstantiate(&ctx->gexec[slot], graph, 0);
    cudaGraphDestroy(graph);
    if (e2 != cudaSuccess) { ctx->gexec[slot] = nullptr; ctx->sw_graph = 0; ctx->launches = l0; cudaGetLastError(); return launch_range_impl(ctx, 0, nf, d_pts, has_intensity, s, false, 0); }
    ctx->glaunches[slot] = ctx->launches - l0;
    ctx->launches = l0;
    have = key;
  }
  CU_TRY(cudaGraphLaunch(ctx->gexec[slot], s));
  ctx->launches += ctx->glaunches[slot];
  ctx->last_pts = d_pts;
  ctx->last_stream = s;
  return PWPP_OK;
}

// Optional sub-batching of a big call (PWPP_SUBBATCH_POINTS=n: consecutive launch sequences of at most n points).
// Off by default: each persistent fit kernel already fills the GPU, so splitting a call only adds tails.
long long subbatch_points() {
  static long long v = [] {
    const char* e = std::getenv("PWPP_SUBBATCH_POINTS");
    return e ? std::atoll(e) : (1LL << 62);   // default: one sequence per call
  }();
  return v;
}

// Launches the frames [f0, f1) of the prepared call: one range per run they overlap (stream order serialises the runs).
// *r is the first run that may overlap; calls with increasing f0 pass the same cursor.
int launch_runs(pwpp_ctx* ctx, int f0, int f1, size_t* r, const float4* d_pts, int has_intensity, cudaStream_t s, bool prof) {
  const std::vector<int>& runs = ctx->runs;
  while (*r + 2 < runs.size() && runs[*r + 1] <= f0) ++*r;
  for (size_t q = *r; q + 1 < runs.size() && runs[q] < f1; ++q) {
    const int a = std::max(f0, runs[q]), b = std::min(f1, runs[q + 1]);
    if (a >= b) continue;
    const int rc = launch_range(ctx, a, b - a, d_pts, has_intensity, s, prof);
    if (rc) return rc;
  }
  return PWPP_OK;
}

// Launches the whole prepared call on stream s.
int launch_call(pwpp_ctx* ctx, int nframes, const float4* d_pts, int has_intensity, cudaStream_t s) {
  int rc = PWPP_OK;
  size_t r = 0;
  // per-stage timing covers one launch sequence: a call of several runs is launched, but not timed
  if (ctx->profiling) return launch_runs(ctx, 0, nframes, &r, d_pts, has_intensity, s, ctx->runs.size() == 2);
  const long long cap = subbatch_points();
  int f0 = 0;
  while (f0 < nframes) {
    int f1 = f0 + 1;
    while (f1 < nframes && ctx->pt_off[f1 + 1] - ctx->pt_off[f0] <= cap) ++f1;
    rc = launch_runs(ctx, f0, f1, &r, d_pts, has_intensity, s, false);
    if (rc) return rc;
    f0 = f1;
  }
  return PWPP_OK;
}

int run_path(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float4* d_pts, int has_intensity, cudaStream_t s) {
  const int rc = prepare_call(ctx, nframes, streams, s);
  if (rc) return rc;
  return launch_call(ctx, nframes, d_pts, has_intensity, s);
}

// A page-locked host buffer, which the upload can read by DMA straight from.
bool page_locked(const void* p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) == cudaSuccess) return attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  return false;
}

// The host-input pipeline of pwpp_estimate_host(_streams) and pwpp_estimate_host_records, after their argument checks, from
// the freeze check to last_time_us. Chunks of frames flow through three streams: H2D of chunk k+1 | kernels of chunk k | D2H
// of chunk k-1. The caller supplies only what is its own: tables(&recs) reserves and fills its tables once the previous call
// is no longer in flight, before the call is prepared, and names its record table (NULL: none); stage(f0, f1, s_in) puts
// frames [f0, f1) into ctx->d_in on the upload stream s_in.
template <typename Tables, typename Stage>
int host_pipeline(pwpp_ctx* ctx, int nframes, const int32_t* streams, const int64_t* n, int has_intensity, Tables tables, Stage stage) {
  int rc = check_frozen(ctx, nframes, n, true);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  ctx->pt_off.assign(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) ctx->pt_off[f + 1] = ctx->pt_off[f] + n[f];
  const long long total = ctx->pt_off[nframes];
  cudaStream_t s = ctx->stream, s_in = ctx->stream_h2d, s_out = ctx->stream_d2h;
  ctx->call_times_valid = false;
  // the staging buffers of the previous call must not be in flight any more (nor a device-input call on a caller's stream)
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(s));
  CU_TRY(cudaStreamSynchronize(s_in));
  CU_TRY(cudaStreamSynchronize(s_out));
  CU_TRY(ctx->d_in.reserve((size_t) std::max<long long>(total, 1)));
  const RecordFrame* recs = nullptr;
  rc = tables(&recs);
  if (rc) return rc;
  rc = prepare_call(ctx, nframes, streams, s, recs);
  if (rc) return rc;
  CU_TRY(ctx->h_out_idx.reserve((size_t) std::max<long long>(total, 1)));
  CU_TRY(ctx->h_counts.reserve((size_t) 3 * nframes));
  // ~64 MB of points per chunk keeps every stage busy without delaying the first kernels
  int chunk_frames = nframes;
  if (nframes > 1 && total > 0) {
    const long long per_frame = std::max<long long>(1, total / nframes);
    chunk_frames = (int) std::min<long long>(nframes, std::max<long long>(1, (4LL << 20) / per_frame));
  }
  const int nchunks = (nframes + chunk_frames - 1) / chunk_frames;
  // a call that is a single chunk has nothing to pipeline: copies and kernels share one stream (no cross-stream event hops
  // on the critical path of a one-frame call) and four events bracket its three phases (pwpp_call_times_us)
  const bool one_stream = (nchunks == 1);
  if (one_stream) { s_in = s; s_out = s; CU_TRY(cudaEventRecord(ctx->ev_begin, s)); }
  // the launch ranges are the pipeline chunks cut at the run boundaries; per-stage timing needs one range per call
  const bool prof = ctx->profiling && nchunks == 1 && ctx->runs.size() == 2;
  size_t run_cursor = 0;
  for (int k = 0; k < nchunks; ++k) {
    const int f0 = k * chunk_frames, f1 = std::min(nframes, f0 + chunk_frames);
    rc = stage(f0, f1, s_in);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ctx->ev0, s_in));
    if (!one_stream) CU_TRY(cudaStreamWaitEvent(s, ctx->ev0, 0));
    rc = launch_runs(ctx, f0, f1, &run_cursor, ctx->d_in.p, has_intensity, s, prof);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ctx->ev1, s));
    if (!one_stream) CU_TRY(cudaStreamWaitEvent(s_out, ctx->ev1, 0));
    const long long o0 = ctx->pt_off[f0], o1 = ctx->pt_off[f1];
    if (f0 == 0 && f1 == nframes) {   // the three count rows are one contiguous block when the chunk covers the whole call
      CU_TRY(cudaMemcpyAsync(ctx->h_counts.p, ctx->d_counts.p, (size_t) 3 * nframes * sizeof(int), cudaMemcpyDeviceToHost, s_out));
    } else {
      for (int q = 0; q < 3; ++q)
        CU_TRY(cudaMemcpyAsync(ctx->h_counts.p + (size_t) q * nframes + f0, ctx->d_counts.p + (size_t) q * nframes + f0,
                               (size_t) (f1 - f0) * sizeof(int), cudaMemcpyDeviceToHost, s_out));
    }
    if (o1 > o0) CU_TRY(cudaMemcpyAsync(ctx->h_out_idx.p + o0, ctx->d_out_idx.p + o0, (size_t) (o1 - o0) * sizeof(int), cudaMemcpyDeviceToHost, s_out));
  }
  if (one_stream) CU_TRY(cudaEventRecord(ctx->ev_end, s));
  CU_TRY(cudaStreamSynchronize(s_out));
  CU_TRY(cudaStreamSynchronize(s));
  ctx->call_times_valid = one_stream;
  ctx->counts_fetched = true;
  ctx->idx_fetched = true;
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

// The device-input calls after their argument checks: the freeze check of frames of n[f] points, the frame offsets
// (ctx->pt_off), the stream order and, with_input, the ctx's input buffer; body(s) then enqueues the call on its stream s.
template <typename Body>
int device_call(pwpp_ctx* ctx, int nframes, const int64_t* n, bool with_input, void* cuda_stream, Body body) {
  int rc = check_frozen(ctx, nframes, n, with_input);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  ctx->pt_off.assign(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) ctx->pt_off[f + 1] = ctx->pt_off[f] + n[f];
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  // work buffers are reused stream-ordered: a call on a different stream than the previous one waits for it
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  if (!ctx->last_stream && s != ctx->stream) CU_TRY(cudaStreamSynchronize(ctx->stream));   // resets issued before the first call ran on the ctx's own stream
  if (with_input) CU_TRY(ctx->d_in.reserve((size_t) std::max<long long>(ctx->pt_off[nframes], 1)));
  rc = body(s);
  if (rc) return rc;
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

int check_frame(pwpp_ctx* ctx, int f) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (f < 0 || f >= ctx->last_nframes) return fail(PWPP_ERR_INVALID_ARG, "frame index outside the last estimate call");
  return PWPP_OK;
}

// The last bound call's point offsets (the device scan of its accepted counts) into the host description of the last call, and
// with a stream table the sets its frames ran with.
int fetch_offsets(pwpp_ctx* ctx) {
  if (ctx->last_call < 0 || ctx->off_fetched) return PWPP_OK;
  int rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = ctx->last_nframes;
  ctx->pt_off.assign(nf + 1, 0);
  CU_TRY(cudaMemcpyAsync(ctx->pt_off.data(), ctx->d_pt_off.p, (size_t) (nf + 1) * sizeof(long long), cudaMemcpyDeviceToHost, ctx->last_stream));
  if (ctx->sets_on_device) {
    ctx->frame_set.assign(nf, 0);
    CU_TRY(cudaMemcpyAsync(ctx->frame_set.data(), ctx->d_pset.p, (size_t) nf * sizeof(int), cudaMemcpyDeviceToHost, ctx->last_stream));
  }
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->last_total = ctx->pt_off[nf];
  ctx->off_fetched = true;
  return PWPP_OK;
}

int fetch_counts(pwpp_ctx* ctx) {
  if (ctx->counts_fetched) return PWPP_OK;
  int rc = fetch_offsets(ctx);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(ctx->h_counts.reserve((size_t) 3 * ctx->last_nframes));
  CU_TRY(cudaMemcpyAsync(ctx->h_counts.p, ctx->d_counts.p, (size_t) 3 * ctx->last_nframes * sizeof(int), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->counts_fetched = true;
  return PWPP_OK;
}
int fetch_indices(pwpp_ctx* ctx) {
  if (ctx->idx_fetched) return PWPP_OK;
  int rc = fetch_counts(ctx);
  if (rc) return rc;
  CU_TRY(ctx->h_out_idx.reserve((size_t) std::max<long long>(ctx->last_total, 1)));
  if (ctx->last_total > 0)
    CU_TRY(cudaMemcpyAsync(ctx->h_out_idx.p, ctx->d_out_idx.p, (size_t) ctx->last_total * sizeof(int), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->idx_fetched = true;
  return PWPP_OK;
}
int fetch_patches(pwpp_ctx* ctx) {
  if (ctx->patches_fetched) return PWPP_OK;
  int rc = fetch_counts(ctx);
  if (rc) return rc;
  const size_t n = (size_t) ctx->last_nframes * ctx->gs.nbs * 3;
  CU_TRY(ctx->h_centers.reserve(n));
  CU_TRY(ctx->h_normals.reserve(n));
  CU_TRY(cudaMemcpyAsync(ctx->h_centers.p, ctx->d_centers.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaMemcpyAsync(ctx->h_normals.p, ctx->d_normals.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->patches_fetched = true;
  return PWPP_OK;
}

inline int frame_n(const pwpp_ctx* ctx, int f) { return (int) (ctx->pt_off[f + 1] - ctx->pt_off[f]); }
// fetched count of frame f: q = 0 ground points, 1 patches, 2 dropped points
inline int count_of(const pwpp_ctx* ctx, int q, int f) { return ctx->h_counts.p[(size_t) q * ctx->last_nframes + f]; }
// frame f's ground or non-ground list in the fetched counts: its start inside the frame's region (the non-ground list follows
// the ground list) and its length (the dropped points are in neither)
struct FrameList { int start, count; };
inline FrameList frame_list(const pwpp_ctx* ctx, int f, bool ground) {
  const int ng = count_of(ctx, 0, f);
  return ground ? FrameList{0, ng} : FrameList{ng, frame_n(ctx, f) - ng - count_of(ctx, 2, f)};
}

}  // namespace

extern "C" {

void pwpp_params_default(pwpp_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->verbose = 0; p->enable_RNR = 1; p->enable_RVPF = 1; p->enable_TGR = 1;            // patchworkpp.h:80-83
  p->num_iter = 3; p->num_lpr = 20; p->num_min_pts = 10; p->num_zones = 4; p->num_rings_of_interest = 4;  // :85-89
  p->RNR_ver_angle_thr = -15.0; p->RNR_intensity_thr = 0.2;                             // :91-92
  p->sensor_height = 1.723; p->th_seeds = 0.125; p->th_dist = 0.125; p->th_seeds_v = 0.25; p->th_dist_v = 0.1;  // :94-98
  p->max_range = 80.0; p->min_range = 2.7; p->uprightness_thr = 0.707; p->adaptive_seed_selection_margin = -1.2;  // :99-102
  p->intensity_thr = 0.0;
  const int sectors[4] = {16, 32, 54, 32}, rings[4] = {2, 4, 4, 4};                     // :104-105
  for (int k = 0; k < 4; ++k) { p->num_sectors_each_zone[k] = sectors[k]; p->num_rings_each_zone[k] = rings[k]; p->elevation_thr[k] = 0; p->flatness_thr[k] = 0; }
  p->max_flatness_storage = 1000; p->max_elevation_storage = 1000;                      // :107-108
}

const char* pwpp_last_error(void) { return g_last_error.c_str(); }
int pwpp_abi_version(void) { return PWPP_ABI_VERSION; }
int pwpp_num_bins(const pwpp_ctx* ctx) { return ctx ? ctx->gs.nbs : 0; }
int pwpp_stream_num_bins(const pwpp_ctx* ctx, int s) {
  if (!ctx || s < 0 || s >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad stream index");
  return ctx->gs.g[ctx->stream_set[s]].nbins;
}
int pwpp_stream_set(const pwpp_ctx* ctx, int s) {
  if (!ctx || s < 0 || s >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad stream index");
  return ctx->stream_set[s];
}

// The context of pwpp_create and pwpp_create_sets: sets and stream_set (NULL: every stream on set 0) are validated.
static int create_impl(const pwpp_params* sets, int num_sets, const int32_t* stream_set, int device, int num_streams, int64_t max_points_per_frame,
                       pwpp_ctx** out) {
  int rc = PWPP_OK;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(PWPP_ERR_NO_DEVICE, std::string("no CUDA device available (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") +
                                        "); this library has no CPU path");
  if (device < 0 || device >= ndev) return fail(PWPP_ERR_INVALID_ARG, "device index out of range");
  pwpp_ctx* ctx = new pwpp_ctx();
  ctx->device = device;
  ctx->num_streams = num_streams;
  ctx->identity.resize(num_streams);
  for (int i = 0; i < num_streams; ++i) ctx->identity[i] = i;
  ctx->last_pos.assign(num_streams, -1);
  ctx->stream_set.assign(num_streams, 0);
  if (stream_set) ctx->stream_set.assign(stream_set, stream_set + num_streams);
  ctx->num_sets = num_sets;
  ctx->set_params.assign(sets, sets + num_sets);
  ctx->gs.nbs = 0;
  int max_sectors = 0;
  for (int k = 0; k < num_sets; ++k) {
    build_geometry(sets[k], ctx->gs.g[k], ctx->aps.a[k], ctx->set_fast[k]);
    ctx->set_hcap[k] = history_cap(ctx->gs.g[k], ctx->aps.a[k]);
    ctx->gs.nbs = std::max(ctx->gs.nbs, ctx->gs.g[k].nbins);
    ctx->hist_stride = std::max(ctx->hist_stride, ctx->set_hcap[k]);
    for (int z = 0; z < 4; ++z) max_sectors = std::max(max_sectors, ctx->gs.g[k].num_sectors[z]);
  }
  ctx->sw_serial_fit = env_int("PWPP_SERIAL_FIT", 0, 0, 1) != 0;       // diagnostic: the fit kernels one after another on the call's stream
  ctx->sw_front = env_int("PWPP_FRONT", PWPP_FRONT_DEFAULT, 0, 1);        // 1: cluster-per-frame front end, 0: k_bin_hist + k_bin_scan + k_scatter
  ctx->sw_patch = env_int("PWPP_FIT_PATCH", PWPP_FIT_PATCH_DEFAULT, 0, 1);   // 1: patches above 512 points on k_fit_patch
  ctx->sw_graph = env_int("PWPP_GRAPH", 1, 0, 1);
  ctx->small_call_frames = env_int("PWPP_SMALL_CALL", PWPP_SMALL_CALL_DEFAULT, 0, 64);   // calls of at most this many frames take the small-call kernels (0: never)
  ctx->nbp = ((ctx->gs.nbs + PW_NUM_PSEUDO + 31) / 32) * 32;
  ctx->max_sectors = max_sectors;
#define CU_TRY_CTX(expr)                                                                                  \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess) {                                                                              \
      std::string m = std::string(#expr) + ": " + cudaGetErrorString(_e);                                 \
      pwpp_destroy(ctx);                                                                                  \
      return fail(PWPP_ERR_CUDA, m);                                                                      \
    }                                                                                                     \
  } while (0)
  CU_TRY_CTX(cudaSetDevice(device));
  CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->stream_h2d, cudaStreamNonBlocking));
  CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->stream_d2h, cudaStreamNonBlocking));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev0));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev1));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev_begin));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev_end));
  for (int i = 0; i <= PWPP_NUM_STAGES; ++i) CU_TRY_CTX(cudaEventCreate(&ctx->stage_ev[i]));
  for (int i = 0; i < 2; ++i) CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->tab_ev[i], cudaEventDisableTiming));
  CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  for (int q = 0; q < NUM_SIDE; ++q) {
    CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->side[q], cudaStreamNonBlocking));
    CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->ev_fit[q], cudaEventDisableTiming));
    CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->ev_join[q], cudaEventDisableTiming));
  }
  CU_TRY_CTX(ctx->d_states.reserve(num_streams));
  CU_TRY_CTX(ctx->d_states_init.reserve(num_streams));
  {
    std::vector<StreamState> v(num_streams);
    for (int i = 0; i < num_streams; ++i) init_state(sets[ctx->stream_set[i]], v[i]);   // the constructor state of the stream's set
    CU_TRY_CTX(cudaMemcpy(ctx->d_states_init.p, v.data(), v.size() * sizeof(StreamState), cudaMemcpyHostToDevice));
  }
  CU_TRY_CTX(ctx->d_hist.reserve((size_t) num_streams * 2 * 4 * ctx->hist_stride));
  // history samples past a stream's counts are never read by the kernels, but pwpp_export_state copies whole rows: zeroed, a
  // blob holds no bytes of whatever the allocation held before
  CU_TRY_CTX(cudaMemset(ctx->d_hist.p, 0, (size_t) num_streams * 2 * 4 * ctx->hist_stride * sizeof(double)));
  {
    std::vector<int> hcap(num_streams);
    for (int i = 0; i < num_streams; ++i) hcap[i] = ctx->set_hcap[ctx->stream_set[i]];
    CU_TRY_CTX(ctx->d_stream_hcap.reserve(num_streams));
    CU_TRY_CTX(cudaMemcpy(ctx->d_stream_hcap.p, hcap.data(), hcap.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU_TRY_CTX(ctx->d_claim.reserve(num_streams));
    CU_TRY_CTX(cudaMemset(ctx->d_claim.p, 0xff, (size_t) num_streams * sizeof(int)));
  }
  CU_TRY_CTX(ctx->d_counts.reserve((size_t) 3 * num_streams));
  CU_TRY_CTX(ctx->d_wq_ctr.reserve(2 * NUM_CLASSES + 2 * ORD_NUM_HEADS));
  CU_TRY_CTX(ctx->d_ox_counts.reserve(OX_NUM_STATS));
  CU_TRY_CTX(cudaMemset(ctx->d_ox_counts.p, 0, OX_NUM_STATS * sizeof(unsigned long long)));
  {
    cudaDeviceProp prop;
    CU_TRY_CTX(cudaGetDeviceProperties(&prop, device));
    // Fit kernel of every patch-size class:
    //   S  <= 64      k_fit_resident: 8 lanes x 8 register slots per patch
    //   M  <= 512     k_fit_warp, patch staged in shared memory, plane + moment sums in shared memory, 3 CTAs/SM
    //                 Instruction-fetch sensitive (125 KB of code): the passes take TWO rows per batch, the LPR scans two loads in
    //                 flight (more rows per batch or more loads in flight were slower).
    //   L1 <= 2048    k_fit_warp, x, y, z staged in 24 KB of shared memory per warp: one CTA of 8 warps per SM, so the plane stays
    //                 in registers and the R-VPF round is fused with the R-GPF seed fit (profiles/h100_fit_l1.jsonl)
    //                 PWPP_FIT_PATCH=1 (and calls of <= 4 frames): k_fit_patch, one patch per CTA of 4 / 8 / 16 warps held in registers
    //   L2 <= 4096    k_fit_cta, per-patch state in shared memory, 4 CTAs/SM
    //   L3 <= 8192    k_fit_cta, 2 CTAs/SM
    //   X  >  8192    k_fit_big (dense sensors)
    const size_t sm_m = FITW_SMEM_M, sm_l2 = 3 * 4096 * sizeof(float), sm_l3 = 3 * 8192 * sizeof(float);
    ctx->fit[0] = {k_fit_resident<8, 8, 0, 2>, 0, FIT_THREADS, 0};
    ctx->fit[1] = {k_fit_warp<true, 1, 1, 2, 3, false, true>, 0, FITW_WARPS * 32, sm_m};
    ctx->fit[2] = {k_fit_warp<true, 2, 2, 2, 1, true, false, true>, 0, FITW_WARPS * 32, FITW_SMEM_L1};
    ctx->fit[3] = {k_fit_cta<4096, 3, 4, 8, true, true>, 0, FIT_THREADS, sm_l2};
    ctx->fit[4] = {k_fit_cta<8192, 4, 2, 8, true>, 0, FIT_THREADS, sm_l3};
    ctx->fit[5] = {k_fit_big<16, 1, true>, 0, 512, 0};
    if (ctx->sw_patch) {
      ctx->fit[2] = {k_fit_patch<4, 4, 2>, 0, 4 * 32, (size_t) 4 * FP_STG * sizeof(float4)};
      ctx->fit[3] = {k_fit_patch<8, 2, 3>, 0, 8 * 32, (size_t) 8 * FP_STG * sizeof(float4)};
      ctx->fit[4] = {k_fit_patch<16, 1, 4>, 0, 16 * 32, (size_t) 16 * FP_STG * sizeof(float4)};
    }
    for (int c = 0; c < NUM_CLASSES; ++c) ctx->fit_small[c] = ctx->fit[c];
    ctx->fit_small[2] = {k_fit_patch<4, 4, 2>, 0, 4 * 32, (size_t) 4 * FP_STG * sizeof(float4)};
    ctx->fit_small[3] = {k_fit_patch<8, 2, 3>, 0, 8 * 32, (size_t) 8 * FP_STG * sizeof(float4)};
    ctx->fit_small[4] = {k_fit_patch<16, 1, 4>, 0, 16 * 32, (size_t) 16 * FP_STG * sizeof(float4)};
    for (int c = 0; c < 2 * NUM_CLASSES; ++c) {
      FitLaunch& k = c < NUM_CLASSES ? ctx->fit[c] : ctx->fit_small[c - NUM_CLASSES];
      if (k.smem > 0) CU_TRY_CTX(raise_smem_limit(k.fn, k.smem));
      int per_sm = 1;
      CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.fn, k.threads, k.smem));
      k.grid = std::max(1, per_sm) * prop.multiProcessorCount;
    }
    {
      typedef void (*OrdKernel)(const float4*, WorkQueues, int*, int*);
      const OrdKernel fn[ORD_NUM_HEADS] = {k_order_cta<512, 5>, k_order_cta<512, 4>, k_order_cta<256, 3>, k_order_cta<128, 2>, k_order_warp};
      const int th[ORD_NUM_HEADS] = {512, 512, 256, 128, ORD_WARP_THREADS};
      for (int q = 0; q < ORD_NUM_HEADS; ++q) {
        const size_t sm = q < 4 ? ord_cta_smem_bytes(th[q]) : 0;
        if (sm > 48 * 1024) CU_TRY_CTX(raise_smem_limit(fn[q], sm));
        int per_sm = 1;
        CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn[q], th[q], sm));
        ctx->order_k[q].grid = std::max(1, per_sm) * prop.multiProcessorCount;
        ctx->order_k[q].threads = th[q];
        ctx->order_k[q].smem = sm;
      }
      typedef void (*OxKernel)(const float4*, WorkQueues, int*, int*, unsigned*, unsigned long long*);
      const OxKernel fx[4] = {k_order_exact_big<5>, k_order_exact_big<4>, k_order_exact_big<3>, k_order_exact_big<2>};
      for (int q = 0; q < ORD_NUM_HEADS; ++q) {
        const size_t sm = q < 4 ? 0 : ox_warp_smem_bytes();
        int per_sm = 1;
        if (q < 4) {
          CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fx[q], OX_WARP_THREADS, 0));
        } else {
          if (sm > 48 * 1024) CU_TRY_CTX(raise_smem_limit(k_order_exact_warp, sm));
          CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_order_exact_warp, OX_WARP_THREADS, sm));
        }
        ctx->exact_k[q].grid = std::max(1, per_sm) * prop.multiProcessorCount;
        ctx->exact_k[q].threads = OX_WARP_THREADS;
        ctx->exact_k[q].smem = sm;
      }
    }
    // reference arithmetic: one CTA per patch, 128 threads up to 512 points, 256 up to 4096 and 512 above, shared capacity 512 / 2048
    // points (larger patches in the global scratch)
    {
      const size_t sm_s = ref32_smem_bytes(R32_SMALL_CAP), sm_b = ref32_smem_bytes(R32_BIG_CAP);
      ctx->fit_ref32[0] = {k_fit_ref32<0, 128, R32_SMALL_CAP>, 0, 128, sm_s};
      ctx->fit_ref32[1] = {k_fit_ref32<1, 128, R32_SMALL_CAP>, 0, 128, sm_s};
      ctx->fit_ref32[2] = {k_fit_ref32<2, 256, R32_BIG_CAP>, 0, 256, sm_b};
      ctx->fit_ref32[3] = {k_fit_ref32<3, 256, R32_BIG_CAP>, 0, 256, sm_b};
      ctx->fit_ref32[4] = {k_fit_ref32<4, 512, R32_BIG_CAP>, 0, 512, sm_b};
      ctx->fit_ref32[5] = {k_fit_ref32<5, 512, R32_BIG_CAP>, 0, 512, sm_b};
      for (Ref32Launch& k : ctx->fit_ref32) {
        if (k.smem > 48 * 1024) CU_TRY_CTX(raise_smem_limit(k.fn, k.smem));
        int per_sm = 1;
        CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.fn, k.threads, k.smem));
        k.grid = std::max(1, per_sm) * prop.multiProcessorCount;
      }
    }
    const size_t gle_smem = gle_smem_bytes(max_sectors);
    if (gle_smem > 48 * 1024) { CU_TRY_CTX(raise_smem_limit(k_gle<false>, gle_smem)); CU_TRY_CTX(raise_smem_limit(k_gle<true>, gle_smem)); }
  }
  {
    const size_t scat = (size_t) (CHUNK_THREADS / 32) * ctx->nbp * sizeof(unsigned int);
    if (scat > 48 * 1024) CU_TRY_CTX(raise_smem_limit(k_scatter<false, 4>, scat));
    const size_t sm_f = front_cluster_smem_bytes(ctx->nbp, FC_THREADS), sm_fd = front_cluster_smem_bytes(ctx->nbp, FC_THREADS_DENSE);
    if (sm_f > 220 * 1024) ctx->sw_front = 0;   // (thousands of bins: the per-warp count tables no longer fit next to the tiles)
    ctx->front_dense_ok = sm_fd <= 220 * 1024;
    if (ctx->sw_front) {
      CU_TRY_CTX(raise_smem_limit(k_front_cluster<true, CLS_L2_MAX, FC_THREADS>, sm_f));
      CU_TRY_CTX(raise_smem_limit(k_front_cluster<false, CLS_L2_MAX, FC_THREADS>, sm_f));
      if (ctx->front_dense_ok) {
        CU_TRY_CTX(raise_smem_limit(k_front_cluster<true, CLS_L2_MAX, FC_THREADS_DENSE>, sm_fd));
        CU_TRY_CTX(raise_smem_limit(k_front_cluster<false, CLS_L2_MAX, FC_THREADS_DENSE>, sm_fd));
      }
    }
  }
  *out = ctx;
  rc = pwpp_reset_all(ctx);
  if (rc) { pwpp_destroy(ctx); *out = nullptr; return rc; }
  CU_TRY_CTX(cudaStreamSynchronize(ctx->stream));   // the initial state is in place before any caller stream can read it
  if (max_points_per_frame > 0) {
    const size_t tot = (size_t) max_points_per_frame * num_streams;
    CU_TRY_CTX(ctx->d_bin_ids.reserve(tot));
    CU_TRY_CTX(ctx->d_sorted.reserve(tot));
    CU_TRY_CTX(ctx->d_part.reserve(tot));
    CU_TRY_CTX(ctx->d_out_idx.reserve(tot));
  }
#undef CU_TRY_CTX
  return PWPP_OK;
}

static int check_create_args(int num_streams, int64_t max_points_per_frame, pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  if (num_streams < 1 || num_streams > 65535) return fail(PWPP_ERR_INVALID_ARG, "num_streams must be in [1,65535]");
  if (max_points_per_frame < 0) return fail(PWPP_ERR_INVALID_ARG, "max_points_per_frame < 0");
  return PWPP_OK;
}

int pwpp_create(const pwpp_params* params, int device, int num_streams, int64_t max_points_per_frame, pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  int rc = validate_params(params);
  if (rc) return rc;
  rc = check_create_args(num_streams, max_points_per_frame, out);
  if (rc) return rc;
  return create_impl(params, 1, nullptr, device, num_streams, max_points_per_frame, out);
}

int pwpp_create_sets(const pwpp_params* sets, int num_sets, const int32_t* stream_set, int device, int num_streams, int64_t max_points_per_frame,
                     pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  if (num_sets < 1 || num_sets > PWPP_MAX_PARAM_SETS)
    return fail(PWPP_ERR_INVALID_ARG, "num_sets must be in [1, " + std::to_string(PWPP_MAX_PARAM_SETS) + "], got " + std::to_string(num_sets));
  if (!sets) return fail(PWPP_ERR_INVALID_ARG, "sets is NULL");
  for (int k = 0; k < num_sets; ++k) {
    const int rc = validate_params(&sets[k]);
    if (rc) return fail(rc, "parameter set " + std::to_string(k) + ": " + g_last_error);
  }
  int rc = check_create_args(num_streams, max_points_per_frame, out);
  if (rc) return rc;
  if (!stream_set) return fail(PWPP_ERR_INVALID_ARG, "stream_set is NULL");
  for (int i = 0; i < num_streams; ++i)
    if (stream_set[i] < 0 || stream_set[i] >= num_sets)
      return fail(PWPP_ERR_INVALID_ARG, "stream " + std::to_string(i) + " names parameter set " + std::to_string(stream_set[i]) + ", outside [0, num_sets)");
  return create_impl(sets, num_sets, stream_set, device, num_streams, max_points_per_frame, out);
}

void pwpp_destroy(pwpp_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (int i = 0; i <= PWPP_NUM_STAGES; ++i) if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]);
  for (int i = 0; i < 2; ++i) if (ctx->gexec[i]) cudaGraphExecDestroy(ctx->gexec[i]);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  for (int i = 0; i < 2; ++i) if (ctx->tab_ev[i]) cudaEventDestroy(ctx->tab_ev[i]);
  for (int q = 0; q < NUM_SIDE; ++q) { if (ctx->ev_fit[q]) cudaEventDestroy(ctx->ev_fit[q]); if (ctx->ev_join[q]) cudaEventDestroy(ctx->ev_join[q]); if (ctx->side[q]) cudaStreamDestroy(ctx->side[q]); }
  if (ctx->ev_rec_off) cudaEventDestroy(ctx->ev_rec_off);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->ev_begin) cudaEventDestroy(ctx->ev_begin);
  if (ctx->ev_end) cudaEventDestroy(ctx->ev_end);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->stream_h2d) cudaStreamDestroy(ctx->stream_h2d);
  if (ctx->stream_d2h) cudaStreamDestroy(ctx->stream_d2h);
  delete ctx;   // the buffers free themselves, on the device set above
}

int pwpp_reset_stream(pwpp_ctx* ctx, int f) {
  if (!ctx || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad stream index");
  int rc = bind_device(ctx);
  if (rc) return rc;
  cudaStream_t s = ctx->last_stream ? ctx->last_stream : ctx->stream;
  CU_TRY(cudaMemcpyAsync(ctx->d_states.p + f, ctx->d_states_init.p + f, sizeof(StreamState), cudaMemcpyDeviceToDevice, s));
  return PWPP_OK;
}
int pwpp_reset_all(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  cudaStream_t s = ctx->last_stream ? ctx->last_stream : ctx->stream;
  CU_TRY(cudaMemcpyAsync(ctx->d_states.p, ctx->d_states_init.p, (size_t) ctx->num_streams * sizeof(StreamState), cudaMemcpyDeviceToDevice, s));
  return PWPP_OK;
}

void* pwpp_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) { g_last_error = "cudaMallocHost failed"; return nullptr; }
  return p;
}
void pwpp_host_free(void* p) { if (p) cudaFreeHost(p); }

int pwpp_set_profiling(pwpp_ctx* ctx, int enabled) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  ctx->profiling = enabled != 0;
  ctx->stage_valid = false;
  return PWPP_OK;
}
int pwpp_stage_times_ms(pwpp_ctx* ctx, float* ms) {
  if (!ctx || !ms) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (!ctx->stage_valid) return fail(PWPP_ERR_INVALID_ARG, "no profiled estimate call yet (pwpp_set_profiling)");
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaEventSynchronize(ctx->stage_ev[PWPP_NUM_STAGES]));
  for (int i = 0; i < PWPP_NUM_STAGES; ++i) CU_TRY(cudaEventElapsedTime(&ms[i], ctx->stage_ev[i], ctx->stage_ev[i + 1]));
  return PWPP_OK;
}
const char* pwpp_stage_name(int stage) {
  static const char* names[PWPP_NUM_STAGES] = {"k_bin_hist", "k_bin_scan", "k_scatter", "k_fit_S", "k_fit_L3", "k_fit_L2", "k_fit_L1", "k_fit_M", "k_fit_X", "k_gle", "k_emit"};
  return (stage >= 0 && stage < PWPP_NUM_STAGES) ? names[stage] : "";
}
int64_t pwpp_launch_count(const pwpp_ctx* ctx) { return ctx ? ctx->launches : 0; }

// The host path of pwpp_estimate_host and pwpp_estimate_host_streams (stream table checked by the caller).
static int estimate_host_impl(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float* const* pts, const int64_t* n, int cols,
                              int64_t row_stride, int64_t col_stride) {
  if (!pts || !n) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (cols != 3 && cols != 4) return fail(PWPP_ERR_INVALID_ARG, "cols must be 3 or 4 (x,y,z[,intensity])");
  for (int f = 0; f < nframes; ++f)
    if (n[f] < 0 || (n[f] > 0 && !pts[f])) return fail(PWPP_ERR_INVALID_ARG, "bad frame pointer/size");
  const bool packed = (cols == 4 && col_stride == 1 && row_stride == 4);
  bool staged_any = false;
  auto no_tables = [](const RecordFrame**) -> int { return PWPP_OK; };
  auto stage = [&](int f0, int f1, cudaStream_t s_in) -> int {
    const long long total = ctx->pt_off[nframes];
    for (int f = f0; f < f1; ++f) {
      const int64_t cnt = n[f];
      if (cnt == 0) continue;
      if (packed && page_locked(pts[f])) {  // page-locked caller buffer: DMA straight from it (the private copy of H:152 is the device buffer)
        // frames that follow each other in the caller's buffer travel as one copy
        int f_last = f;
        int64_t run = cnt;
        while (f_last + 1 < f1 && n[f_last + 1] > 0 && pts[f_last + 1] == pts[f_last] + n[f_last] * 4) { ++f_last; run += n[f_last]; }
        CU_TRY(cudaMemcpyAsync(ctx->d_in.p + ctx->pt_off[f], pts[f], (size_t) run * sizeof(float4), cudaMemcpyHostToDevice, s_in));
        f = f_last;
        continue;
      }
      if (row_stride == 1 && col_stride == cnt && cnt > 1) {
        // column-major frame (what the Eigen overload hands over): its cols x n floats are one contiguous block; upload it as
        // it is and repack on the device instead of gathering 4 strided columns per point on the host
        if ((size_t) total * 4 > ctx->d_cm.cap) { CU_TRY(cudaStreamSynchronize(s_in)); CU_TRY(ctx->d_cm.reserve((size_t) total * 4)); }
        float* cm = ctx->d_cm.p + (size_t) ctx->pt_off[f] * 4;
        CU_TRY(cudaMemcpyAsync(cm, pts[f], (size_t) cnt * cols * sizeof(float), cudaMemcpyHostToDevice, s_in));
        k_repack_colmajor<<<(unsigned) ((cnt + 255) / 256), 256, 0, s_in>>>(cm, cnt, cols, ctx->d_in.p + ctx->pt_off[f]);
        ++ctx->launches;
        continue;
      }
      if (!staged_any) { CU_TRY(ctx->h_in.reserve((size_t) std::max<long long>(total, 1))); staged_any = true; }
      float4* dst = ctx->h_in.p + ctx->pt_off[f];
      const float* src = pts[f];
      if (packed) {
        std::memcpy(dst, src, (size_t) cnt * sizeof(float4));
      } else {
        for (int64_t i = 0; i < cnt; ++i) {
          const float* r = src + i * row_stride;
          dst[i] = make_float4(r[0], r[col_stride], r[2 * col_stride], cols == 4 ? r[3 * col_stride] : 0.f);
        }
      }
      CU_TRY(cudaMemcpyAsync(ctx->d_in.p + ctx->pt_off[f], dst, (size_t) cnt * sizeof(float4), cudaMemcpyHostToDevice, s_in));
    }
    return PWPP_OK;
  };
  return host_pipeline(ctx, nframes, streams, n, cols == 4 ? 1 : 0, no_tables, stage);
}

int pwpp_estimate_host(pwpp_ctx* ctx, int nframes, const float* const* pts, const int64_t* n, int cols, int64_t row_stride, int64_t col_stride) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (nframes < 1 || nframes > ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, num_streams]");
  return estimate_host_impl(ctx, nframes, ctx->identity.data(), pts, n, cols, row_stride, col_stride);
}

int pwpp_estimate_host_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float* const* pts, const int64_t* n, int cols,
                               int64_t row_stride, int64_t col_stride) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const int rc = check_streams(ctx, nframes, streams);
  if (rc) return rc;
  return estimate_host_impl(ctx, nframes, streams, pts, n, cols, row_stride, col_stride);
}

// The frame sizes of a device-input call's offsets, which must be non-decreasing.
static int offset_sizes(int nframes, const int64_t* h_offsets, int64_t* sizes) {
  for (int f = 0; f < nframes; ++f) {
    sizes[f] = h_offsets[f + 1] - h_offsets[f];
    if (sizes[f] < 0) return fail(PWPP_ERR_INVALID_ARG, "offsets must be non-decreasing");
  }
  return PWPP_OK;
}

// The device path of pwpp_estimate_device and pwpp_estimate_device_streams (stream table checked by the caller).
static int estimate_device_impl(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* d_pts, const int64_t* h_offsets, int has_intensity,
                                void* cuda_stream) {
  if (!h_offsets) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  std::vector<int64_t> sizes(nframes);
  int rc = offset_sizes(nframes, h_offsets, sizes.data());
  if (rc) return rc;
  if (h_offsets[nframes] > h_offsets[0] && !d_pts) return fail(PWPP_ERR_INVALID_ARG, "d_pts is NULL");
  return device_call(ctx, nframes, sizes.data(), false, cuda_stream, [&](cudaStream_t s) {
    return run_path(ctx, nframes, streams, (const float4*) d_pts + h_offsets[0], has_intensity, s);
  });
}

int pwpp_estimate_device(pwpp_ctx* ctx, int nframes, const void* d_pts, const int64_t* h_offsets, int has_intensity, void* cuda_stream) {
  if (!ctx || !h_offsets) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (nframes < 1 || nframes > ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, num_streams]");
  return estimate_device_impl(ctx, nframes, ctx->identity.data(), d_pts, h_offsets, has_intensity, cuda_stream);
}

int pwpp_estimate_device_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* d_pts, const int64_t* h_offsets, int has_intensity,
                                 void* cuda_stream) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const int rc = check_streams(ctx, nframes, streams);
  if (rc) return rc;
  return estimate_device_impl(ctx, nframes, streams, d_pts, h_offsets, has_intensity, cuda_stream);
}

int pwpp_estimate_device_xyz(pwpp_ctx* ctx, int nframes, const void* d_xyz, const int64_t* h_offsets, void* cuda_stream) {
  if (!ctx || !h_offsets) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (nframes < 1 || nframes > ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, num_streams]");
  const long long total = h_offsets[nframes] - h_offsets[0];
  if (total < 0 || (total > 0 && !d_xyz)) return fail(PWPP_ERR_INVALID_ARG, "bad offsets / d_xyz is NULL");
  std::vector<int64_t> sizes(nframes);
  const int rc = offset_sizes(nframes, h_offsets, sizes.data());
  if (rc) return rc;
  return device_call(ctx, nframes, sizes.data(), true, cuda_stream, [&](cudaStream_t s) {
    if (total > 0) {
      k_pad_xyz<<<(unsigned) ((total + 255) / 256), 256, 0, s>>>((const float*) d_xyz + 3 * h_offsets[0], total, ctx->d_in.p);
      ++ctx->launches;
    }
    return run_path(ctx, nframes, ctx->identity.data(), ctx->d_in.p, 0, s);
  });
}

// The checks of both records entry points (include/pwpp.h), before anything is allocated or launched.
static int check_records_call(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* n,
                              const pwpp_point_layout* layouts) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = check_streams(ctx, nframes, streams);
  if (rc) return rc;
  std::string msg;
  rc = check_record_layouts(nframes, frames, n, layouts, &msg);
  if (rc) return fail(rc, msg);
  for (int f = 0; f < nframes; ++f)
    if (n[f] > 0x7fffffffLL - CHUNK_PTS) return fail(PWPP_ERR_INVALID_ARG, "frame " + std::to_string(f) + ": frame size out of range");
  return PWPP_OK;
}

// Unpacks frames [f0, f1) of the prepared records call into ctx->d_in on stream s: one launch (none when the frames are empty).
static int unpack_records(pwpp_ctx* ctx, int f0, int f1, const std::vector<RecordFrame>& recs, cudaStream_t s) {
  if (ctx->pt_off[f1] == ctx->pt_off[f0]) return PWPP_OK;
  const long long gx = rec_grid_x(ctx->pt_off.data() + f0, recs.data() + f0, f1 - f0);
  k_unpack_records<<<dim3((unsigned) gx, (unsigned) (f1 - f0)), REC_THREADS, 0, s>>>(ctx->d_rec.p + f0, ctx->d_pt_off.p + f0, ctx->d_in.p);
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  return PWPP_OK;
}

int pwpp_estimate_host_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* n,
                               const pwpp_point_layout* layouts) {
  const int rc = check_records_call(ctx, nframes, streams, frames, n, layouts);
  if (rc) return rc;
  std::vector<long long> raw_off(nframes + 1, 0);   // every frame's records in the upload buffer, 16-byte aligned
  int has_intensity = 0;
  for (int f = 0; f < nframes; ++f) {
    raw_off[f + 1] = raw_off[f] + ((n[f] * layouts[f].point_step + 15) & ~15LL);
    if (layouts[f].offset[3] >= 0) has_intensity = 1;
  }
  std::vector<RecordFrame> recs(nframes);
  auto tables = [&](const RecordFrame** out) -> int {
    CU_TRY(ctx->d_raw.reserve((size_t) std::max<long long>(raw_off[nframes], 16)));
    for (int f = 0; f < nframes; ++f) recs[f] = record_frame(layouts[f], ctx->d_raw.p + raw_off[f]);
    *out = recs.data();
    return PWPP_OK;
  };
  bool staged_any = false;
  // H2D + unpack of a chunk's records
  auto stage = [&](int f0, int f1, cudaStream_t s_in) -> int {
    // a call of several chunks unpacks on the upload stream, and the unpack reads the record table uploaded on the call's stream
    if (f0 == 0 && s_in != ctx->stream) CU_TRY(cudaStreamWaitEvent(s_in, ctx->tab_ev[ctx->tab_cur], 0));
    for (int f = f0; f < f1; ++f) {
      if (n[f] == 0) continue;
      const size_t bytes = (size_t) n[f] * layouts[f].point_step;
      const void* src = frames[f];
      if (!page_locked(src)) {   // pageable: one memcpy into page-locked staging, then DMA
        if (!staged_any) { CU_TRY(ctx->h_raw.reserve((size_t) std::max<long long>(raw_off[nframes], 16))); staged_any = true; }
        std::memcpy(ctx->h_raw.p + raw_off[f], frames[f], bytes);
        src = ctx->h_raw.p + raw_off[f];
      }
      CU_TRY(cudaMemcpyAsync(ctx->d_raw.p + raw_off[f], src, bytes, cudaMemcpyHostToDevice, s_in));
    }
    return unpack_records(ctx, f0, f1, recs, s_in);
  };
  return host_pipeline(ctx, nframes, streams, n, has_intensity, tables, stage);
}

int pwpp_estimate_device_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* d_frames, const int64_t* n,
                                 const pwpp_point_layout* layouts, void* cuda_stream) {
  const int rc = check_records_call(ctx, nframes, streams, d_frames, n, layouts);
  if (rc) return rc;
  return device_call(ctx, nframes, n, true, cuda_stream, [&](cudaStream_t s) {
    std::vector<RecordFrame> recs(nframes);
    int has_intensity = 0;
    for (int f = 0; f < nframes; ++f) {
      recs[f] = record_frame(layouts[f], d_frames[f]);
      if (layouts[f].offset[3] >= 0) has_intensity = 1;
    }
    int rc = prepare_call(ctx, nframes, streams, s, recs.data());
    if (rc) return rc;
    rc = unpack_records(ctx, 0, nframes, recs, s);
    if (rc) return rc;
    return launch_call(ctx, nframes, ctx->d_in.p, has_intensity, s);
  });
}

// ---- the bound call (include/pwpp.h) ----

// Makes bound call k the ctx's last call, run on stream s: the host getters fetch its offsets first (fetch_offsets).
static void make_bound_last(pwpp_ctx* ctx, int k, cudaStream_t s) {
  const pwpp_ctx::Bound& b = ctx->bound[k];
  ctx->last_nframes = b.nf;
  ctx->frame_set = b.frame_set;
  ctx->last_recs.clear();
  ctx->last_pts = ctx->d_in.p;
  ctx->last_stream = s;
  ctx->last_total = 0;
  ctx->last_call = k;
  ctx->sets_on_device = b.d_streams != nullptr;
  ctx->off_fetched = ctx->counts_fetched = ctx->idx_fetched = ctx->patches_fetched = false;
  ctx->rec_gathered = ctx->rec_fetched = false;
  ctx->stage_valid = ctx->call_times_valid = false;
}

int pwpp_bind_call(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* max_n,
                   const pwpp_point_layout* layouts, const int64_t* d_counts) {
  return pwpp_bind_call_actions(ctx, nframes, streams, frames, max_n, layouts, d_counts, nullptr);
}

// The checks of a ring-bound call beyond those of pwpp_bind_call (frames[f] = rings[f].base): the ring of every frame.
static int check_rings(int nframes, const pwpp_scan_ring* rings, const int64_t* max_n, const pwpp_point_layout* layouts) {
  for (int f = 0; f < nframes; ++f) {
    const std::string fr = "frame " + std::to_string(f) + ": ";
    const pwpp_scan_ring& R = rings[f];
    const long long bytes = max_n[f] * layouts[f].point_step;   // (max_n < 2^31 and point_step <= PWPP_MAX_POINT_STEP: no overflow)
    if (!R.d_counts) return fail(PWPP_ERR_INVALID_ARG, fr + "ring d_counts is NULL");
    if (R.num_slots < 1) return fail(PWPP_ERR_INVALID_ARG, fr + "ring num_slots " + std::to_string(R.num_slots) + " < 1");
    if (R.slot_stride < bytes)
      return fail(PWPP_ERR_INVALID_ARG, fr + "ring slot_stride " + std::to_string(R.slot_stride) + " < max_n * point_step = " + std::to_string(bytes));
    // the kernels form base + s * slot_stride in 64 bits: the extent and its end address must not overflow
    const __int128 extent = (__int128) (R.num_slots - 1) * R.slot_stride + bytes;
    if (extent > (__int128) INT64_MAX || (__int128) (uintptr_t) R.base + extent > (__int128) UINTPTR_MAX)
      return fail(PWPP_ERR_INVALID_ARG, fr + "the ring's extent (num_slots - 1) * slot_stride + max_n * point_step overflows");
  }
  return PWPP_OK;
}

// The checks of a packed bind beyond those of pwpp_bind_call (frames[f] = base): the buffer's extent. They run before the records
// checks, so that a NULL base is named as such.
static int check_packed(const void* base, int64_t capacity, const pwpp_point_layout& layout) {
  if (capacity < 0) return fail(PWPP_ERR_INVALID_ARG, "capacity " + std::to_string(capacity) + " < 0");
  if (!base && capacity > 0) return fail(PWPP_ERR_INVALID_ARG, "base is NULL with capacity " + std::to_string(capacity) + " > 0");
  // the kernels form base + lo * point_step in 64 bits: the extent and its end address must not overflow
  const __int128 extent = (__int128) capacity * layout.point_step;
  if (extent > (__int128) INT64_MAX || (__int128) (uintptr_t) base + extent > (__int128) UINTPTR_MAX)
    return fail(PWPP_ERR_INVALID_ARG, "capacity * point_step (" + std::to_string(capacity) + " * " + std::to_string(layout.point_step) + ") overflows");
  return PWPP_OK;
}

// The bind of pwpp_bind_call, pwpp_bind_call_actions, pwpp_bind_call_rings and pwpp_bind_call_packed. rings is NULL except for
// the ring bind, where frames[f] is rings[f].base and d_counts is unused; d_offsets is NULL except for the packed bind, where
// frames[f] is its base, layouts[f] its layout and d_counts is unused.
// With actions: frame f of run r gets scratch slot num_streams + (f - runs[r]) (distinct inside a run), and dep[f] says whether
// its stream has a frame in an earlier run (then a RESET of f waits for that run: k_bound_reset before f's run).
static int bind_call_impl(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* max_n,
                          const pwpp_point_layout* layouts, const int64_t* d_counts, const int32_t* d_actions, const pwpp_scan_ring* rings,
                          const int32_t* d_slots, const int64_t* d_offsets = nullptr, int64_t capacity = 0) {
  int rc = check_records_call(ctx, nframes, streams, frames, max_n, layouts);
  if (rc) return rc;
  if (ctx->bound[ctx->sel].on)
    return fail(PWPP_ERR_INVALID_ARG, "a call is already bound as bound call " + std::to_string(ctx->sel) + " (pwpp_unbind_call releases it)");
  if (!rings && !d_offsets && !d_counts) return fail(PWPP_ERR_INVALID_ARG, "d_counts is NULL");
  if (rings && (rc = check_rings(nframes, rings, max_n, layouts))) return rc;
  pwpp_ctx::Bound b;
  b.nf = nframes;
  b.d_counts = reinterpret_cast<const long long*>(d_counts);
  b.d_slots = d_slots;
  b.d_offsets = reinterpret_cast<const long long*>(d_offsets);
  b.capacity = capacity;
  b.cap_pt_off.assign(nframes + 1, 0);
  b.cap_chunk_off.assign(nframes + 1, 0);
  long long chunks = 0;
  for (int f = 0; f < nframes; ++f) {
    b.cap_pt_off[f + 1] = b.cap_pt_off[f] + max_n[f];
    chunks += (max_n[f] + CHUNK_PTS - 1) / CHUNK_PTS;
    if (chunks > 0x7fffffffLL) return fail(PWPP_ERR_INVALID_ARG, "frame " + std::to_string(f) + ": the capacities exceed 2^31 - 1 chunks of " + std::to_string(CHUNK_PTS) + " points");
    b.cap_chunk_off[f + 1] = (int) chunks;
  }
  std::vector<RecordFrame> recs(nframes);
  for (int f = 0; f < nframes; ++f) {
    recs[f] = record_frame(layouts[f], frames[f]);
    if (layouts[f].offset[3] >= 0) b.has_intensity = 1;
    b.frame_set.push_back(ctx->stream_set[streams[f]]);
  }
  b.recs = recs;
  split_runs(ctx, nframes, streams);
  b.runs = ctx->runs;
  std::vector<int> scratch, dep;
  int slots = 0;   // the longest run
  if (d_actions) {
    b.d_actions = d_actions;
    scratch.resize(nframes);
    dep.resize(nframes);
    std::vector<int> first_run(ctx->num_streams, -1);
    b.reset_run.assign(b.runs.size() - 1, 0);
    for (size_t r = 0; r + 1 < b.runs.size(); ++r) {
      slots = std::max(slots, b.runs[r + 1] - b.runs[r]);
      for (int f = b.runs[r]; f < b.runs[r + 1]; ++f) {
        int& fr = first_run[streams[f]];
        if (fr < 0) fr = (int) r;
        scratch[f] = ctx->num_streams + (f - b.runs[r]);
        dep[f] = fr < (int) r;
        if (dep[f]) b.reset_run[r] = 1;
      }
    }
  }
  if ((rc = check_growth(ctx, slots, nframes, b.cap_pt_off[nframes], chunks))) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  // the buffers may move: whatever the ctx enqueued before has finished with them, and the last call's results end here
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  ctx->last_nframes = 0;
  ctx->last_call = -1;
  if (slots > ctx->scratch_slots) {
    // the streams' states and histories move with their contents; a failed allocation leaves them where they were
    const size_t ns = (size_t) ctx->num_streams + slots;
    CU_TRY(ctx->d_states.grow_keep(ns));
    CU_TRY(ctx->d_hist.grow_keep(ns * 2 * 4 * ctx->hist_stride));
    ctx->scratch_slots = slots;
  }
  if (slots > 0) {
    // a scratch slot starts as a constructor state (empty histories): the empty frames redirected there keep it empty, so
    // k_gle never reads a history sample of a scratch slot
    StreamState s0;
    CU_TRY(cudaMemcpy(&s0, ctx->d_states_init.p, sizeof(StreamState), cudaMemcpyDeviceToHost));
    const std::vector<StreamState> fill(slots, s0);
    CU_TRY(cudaMemcpy(ctx->d_states.p + ctx->num_streams, fill.data(), (size_t) slots * sizeof(StreamState), cudaMemcpyHostToDevice));
  }
  rc = reserve_work(ctx, nframes, b.cap_pt_off[nframes], chunks, true, false);
  if (rc) return rc;
  // the bound call's own buffers: an error from here on frees them with b
  if (d_actions) {
    CU_TRY(b.d_bscratch.reserve(nframes));
    CU_TRY(b.d_bdep.reserve(nframes));
    CU_TRY(b.d_bact.reserve(nframes));
    CU_TRY(cudaMemcpy(b.d_bscratch.p, scratch.data(), (size_t) nframes * sizeof(int), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(b.d_bdep.p, dep.data(), (size_t) nframes * sizeof(int), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemset(b.d_bact.p, 0, (size_t) nframes * sizeof(int)));
  }
  CU_TRY(b.d_bmax.reserve(nframes));
  CU_TRY(b.d_bstream.reserve(nframes));
  CU_TRY(b.d_bpset.reserve(nframes));
  CU_TRY(b.d_bstatus.reserve(nframes));
  CU_TRY(b.d_brec.reserve(nframes));
  CU_TRY(cudaMemcpy(b.d_bmax.p, max_n, (size_t) nframes * sizeof(long long), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(b.d_bstream.p, streams, (size_t) nframes * sizeof(int), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(b.d_bpset.p, b.frame_set.data(), (size_t) nframes * sizeof(int), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(b.d_brec.p, recs.data(), (size_t) nframes * sizeof(RecordFrame), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemset(b.d_bstatus.p, 0, (size_t) nframes * sizeof(int)));
  CU_TRY(b.d_width.reserve(1));
  CU_TRY(cudaMemcpy(b.d_width.p, &nframes, sizeof(int), cudaMemcpyHostToDevice));
  if (rings) {
    std::vector<BoundRing> ring(nframes);
    for (int f = 0; f < nframes; ++f)
      ring[f] = BoundRing{reinterpret_cast<const long long*>(rings[f].d_counts), (long long) rings[f].slot_stride, (int) rings[f].num_slots, 0};
    CU_TRY(b.d_bring.reserve(nframes));
    CU_TRY(b.d_bslot.reserve(nframes));
    CU_TRY(b.d_brun.reserve(nframes));
    CU_TRY(cudaMemcpy(b.d_bring.p, ring.data(), (size_t) nframes * sizeof(BoundRing), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(b.d_brun.p, recs.data(), (size_t) nframes * sizeof(RecordFrame), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemset(b.d_bslot.p, 0xff, (size_t) nframes * sizeof(int)));   // -1: no run yet
  }
  if (d_offsets) {
    CU_TRY(b.d_brun.reserve(nframes));
    CU_TRY(cudaMemcpy(b.d_brun.p, recs.data(), (size_t) nframes * sizeof(RecordFrame), cudaMemcpyHostToDevice));
  }
  CU_TRY(cudaDeviceSynchronize());
  b.on = true;
  ctx->bound[ctx->sel] = std::move(b);
  return PWPP_OK;
}

int pwpp_bind_call_actions(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* max_n,
                           const pwpp_point_layout* layouts, const int64_t* d_counts, const int32_t* d_actions) {
  return bind_call_impl(ctx, nframes, streams, frames, max_n, layouts, d_counts, d_actions, nullptr, nullptr);
}

int pwpp_bind_call_rings(pwpp_ctx* ctx, int nframes, const int32_t* streams, const pwpp_scan_ring* rings, const int64_t* max_n,
                         const pwpp_point_layout* layouts, const int32_t* d_slots, const int32_t* d_actions) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!rings) return fail(PWPP_ERR_INVALID_ARG, "rings is NULL");
  if (!d_slots) return fail(PWPP_ERR_INVALID_ARG, "d_slots is NULL");
  std::vector<const void*> frames(std::max(nframes, 1), nullptr);
  for (int f = 0; f < nframes; ++f) frames[f] = rings[f].base;
  return bind_call_impl(ctx, nframes, streams, frames.data(), max_n, layouts, nullptr, d_actions, rings, d_slots);
}

int pwpp_bind_call_packed(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* base, const pwpp_point_layout* layout,
                          int64_t capacity, const int64_t* max_n, const int64_t* d_offsets, const int32_t* d_actions) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!layout) return fail(PWPP_ERR_INVALID_ARG, "layout is NULL");
  if (!d_offsets) return fail(PWPP_ERR_INVALID_ARG, "d_offsets is NULL");
  const int rc = check_packed(base, capacity, *layout);
  if (rc) return rc;
  std::vector<const void*> frames(std::max(nframes, 1), base);
  std::vector<pwpp_point_layout> layouts(std::max(nframes, 1), *layout);
  return bind_call_impl(ctx, nframes, streams, frames.data(), max_n, layouts.data(), nullptr, d_actions, nullptr, nullptr, d_offsets, capacity);
}

// An enable that changes what a run of bound call b launches, after its width ladder captured the launch sequences.
static int check_no_ladder(const pwpp_ctx::Bound& b, const char* what) {
  if (b.ladder)
    return fail(PWPP_ERR_INVALID_ARG, std::string("the bound call has a width ladder, which captured its launch sequences: enable ") + what +
                                          " before the width ladder (pwpp_bind_width_ladder)");
  return PWPP_OK;
}

// The host-side description launch_range_impl reads for bound call b (direct calls and other bound calls between runs replace it).
static void describe_bound(pwpp_ctx* ctx, const pwpp_ctx::Bound& b) {
  ctx->last_nframes = b.nf;
  ctx->runs = b.runs;
  ctx->frame_set = b.frame_set;
  ctx->sets_on_device = b.d_streams != nullptr;
  ctx->chunk_off = b.cap_chunk_off;
  ctx->pt_off = b.cap_pt_off;
}

// The first kernel of every run of bound call b: its frame table from the counts, actions, slots, offsets and streams.
static int enqueue_bound_table(pwpp_ctx* ctx, pwpp_ctx::Bound& b, cudaStream_t s) {
  const int nf = b.nf;
  const BoundActions A{b.d_actions, b.d_bact.p, b.d_bscratch.p, b.d_bdep.p, ctx->d_states_init.p, ctx->d_states.p};
  const BoundStreams T{b.d_streams, b.d_bread.p, b.d_bclaim.p, b.d_bset_of.p, b.d_bruns.p, (int) b.runs.size() - 1, ctx->num_streams};
  if (b.d_slots) {
    const BoundRings G{b.d_slots, b.d_bslot.p, b.d_bring.p, b.d_brec.p, b.d_brun.p};
    if (b.d_streams)
      k_bound_table_rings_streams<<<1, BT_THREADS, 0, s>>>(nf, b.d_bmax.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p, ctx->d_stream.p,
                                                           ctx->d_pset.p, b.d_bstatus.p, A, G, T);
    else if (b.d_actions)
      k_bound_table_rings_actions<<<1, BT_THREADS, 0, s>>>(nf, b.d_bmax.p, b.d_bstream.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p,
                                                           ctx->d_stream.p, ctx->d_pset.p, b.d_bstatus.p, A, G);
    else
      k_bound_table_rings<<<1, BT_THREADS, 0, s>>>(nf, b.d_bmax.p, b.d_bstream.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p,
                                                   ctx->d_stream.p, ctx->d_pset.p, b.d_bstatus.p, G);
  } else if (b.d_offsets) {
    const BoundPacked P{b.d_offsets, b.capacity, b.d_brec.p, b.d_brun.p};
    if (b.d_streams)
      k_bound_table_packed_streams<<<1, BT_THREADS, 0, s>>>(nf, b.d_bmax.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p, ctx->d_stream.p,
                                                            ctx->d_pset.p, b.d_bstatus.p, A, P, T);
    else if (b.d_actions)
      k_bound_table_packed_actions<<<1, BT_THREADS, 0, s>>>(nf, b.d_bmax.p, b.d_bstream.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p,
                                                            ctx->d_stream.p, ctx->d_pset.p, b.d_bstatus.p, A, P);
    else
      k_bound_table_packed<<<1, BT_THREADS, 0, s>>>(nf, b.d_bmax.p, b.d_bstream.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p,
                                                    ctx->d_stream.p, ctx->d_pset.p, b.d_bstatus.p, P);
  } else if (b.d_streams) {
    k_bound_table_streams<<<1, BT_THREADS, 0, s>>>(nf, b.d_counts, b.d_bmax.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p, ctx->d_stream.p,
                                                   ctx->d_pset.p, b.d_bstatus.p, A, T);
  } else if (b.d_actions) {
    k_bound_table_actions<<<1, BT_THREADS, 0, s>>>(nf, b.d_counts, b.d_bmax.p, b.d_bstream.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p,
                                                   ctx->d_stream.p, ctx->d_pset.p, b.d_bstatus.p, A);
  } else {
    k_bound_table<<<1, BT_THREADS, 0, s>>>(nf, b.d_counts, b.d_bmax.p, b.d_bstream.p, b.d_bpset.p, ctx->d_pt_off.p, ctx->d_chunk_off.p,
                                           ctx->d_stream.p, ctx->d_pset.p, b.d_bstatus.p);
  }
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  return PWPP_OK;
}

// Everything a run of bound call b launches after its table kernel, cut at width w (1 <= w <= nf): the unpack, then per run the
// reset, the launch sequence and the state rows, then the gathers. Every grid is sized from the capacities of positions [0, w).
// A run's positions at or past w (all rejected when the width rule picked w) are launched as a second range of frames with grids
// for empty frames; the gathers keep grid.y = nf, so those frames' counts come from the same code as without a ladder. With
// w = nf this is the launch sequence of a call without a ladder, grids included. The host description must be b's (describe_bound).
static int enqueue_bound_body(pwpp_ctx* ctx, pwpp_ctx::Bound& b, cudaStream_t s, int w) {
  const int nf = b.nf;
  const RecordFrame* recs = (b.d_slots || b.d_offsets) ? b.d_brun.p : b.d_brec.p;   // the record table the unpack and the gathers read
  const long long* cap = b.cap_pt_off.data();
  if (cap[w] > 0) {
    k_unpack_records<<<dim3((unsigned) rec_grid_x(cap, b.recs.data(), w), (unsigned) w), REC_THREADS, 0, s>>>(recs, ctx->d_pt_off.p, ctx->d_in.p);
    ++ctx->launches;
  }
  CU_TRY(cudaGetLastError());
  for (size_t r = 0; r + 1 < b.runs.size(); ++r) {
    const int f0 = b.runs[r], f1 = b.runs[r + 1], cut = std::min(f1, std::max(f0, w));
    // the RESET frames whose stream ran in an earlier run; with a stream table the host cannot know which, so every RESET frame
    // of every later run (its dep is 1) is reset right before its run, from the streams the run read
    if (b.d_actions && (b.d_streams ? r > 0 : b.reset_run[r])) {
      k_bound_reset<<<1, BR_THREADS, 0, s>>>(f0, f1, b.d_bact.p, b.d_bdep.p, b.d_streams ? b.d_bread.p : b.d_bstream.p,
                                             ctx->d_states_init.p, ctx->d_states.p);
      ++ctx->launches;
      CU_TRY(cudaGetLastError());
    }
    if (cut > f0) {
      int chunks = 0;   // the largest ceil(max_n / CHUNK_PTS) of the range
      for (int f = f0; f < cut; ++f) chunks = std::max(chunks, b.cap_chunk_off[f + 1] - b.cap_chunk_off[f]);
      const int rc = launch_range_impl(ctx, f0, cut - f0, ctx->d_in.p, b.has_intensity, s, false, chunks, f0, f1 - f0);
      if (rc) return rc;
    }
    if (f1 > cut) {
      const int rc = launch_range_impl(ctx, cut, f1 - cut, ctx->d_in.p, b.has_intensity, s, false, -1, f0, f1 - f0);
      if (rc) return rc;
    }
    if (b.getters & PWPP_GETTER_STATE) {   // before a later run moves the run's streams
      const int len = f1 - f0;
      if (b.d_streams)
        k_bound_states_streams<<<(len + BS_THREADS - 1) / BS_THREADS, BS_THREADS, 0, s>>>(f0, f1, b.d_bread.p, ctx->num_streams, ctx->d_states.p,
                                                                                          b.d_bstates.p);
      else
        k_bound_states<<<(len + BS_THREADS - 1) / BS_THREADS, BS_THREADS, 0, s>>>(f0, f1, b.d_bstream.p, ctx->d_states.p, b.d_bstates.p);
      ++ctx->launches;
      CU_TRY(cudaGetLastError());
    }
  }
  const long long rec_gx = rec_parts_grid_x(cap, b.recs.data(), w), xyz_gx = xyz_parts_grid_x(cap, w);
  if (b.rec_parts) {   // the record results: both parts' lists are where the runs' k_emit left them
    const int first = b.rec_parts == PWPP_PART_NONGROUND ? 1 : 0, nparts = b.rec_parts == 3 ? 2 : 1;
    k_gather_record_parts<<<dim3((unsigned) rec_gx, (unsigned) nf, (unsigned) nparts), REC_THREADS, 0, s>>>(
        recs, ctx->d_pt_off.p, ctx->d_counts.p, nf, ctx->d_out_idx.p, b.d_bpart_off.p, first, b.d_bground.p, b.d_bnonground.p,
        b.d_rec_counts.p);
    ++ctx->launches;
    CU_TRY(cudaGetLastError());
  }
  if (b.getters & (PWPP_GETTER_GROUND_XYZ | PWPP_GETTER_NONGROUND_XYZ)) {   // the xyz of both lists, from the unpacked points
    const int parts = b.getters & 3, first = parts == PWPP_GETTER_NONGROUND_XYZ ? 1 : 0, nparts = parts == 3 ? 2 : 1;
    k_gather_xyz_parts<<<dim3((unsigned) xyz_gx, (unsigned) nf, (unsigned) nparts), XYZ_THREADS, 0, s>>>(
        ctx->d_in.p, ctx->d_pt_off.p, ctx->d_counts.p, nf, ctx->d_out_idx.p, b.d_bxyz_off.p, first, b.d_bgxyz.p, b.d_bngxyz.p,
        b.d_xyz_counts.p);
    ++ctx->launches;
    CU_TRY(cudaGetLastError());
  }
  if (b.packed_xyz || b.packed_rec) {   // the offsets of both parts from the final counts (one scan for both), then the rows
    k_bound_xyz_offsets<<<1, BT_THREADS, 0, s>>>(nf, ctx->d_pt_off.p, ctx->d_counts.p, b.d_pg_off.p, b.d_png_off.p);
    ++ctx->launches;
    if (b.packed_xyz) {
      const int first = b.packed_xyz == PWPP_PART_NONGROUND ? 1 : 0, nparts = b.packed_xyz == 3 ? 2 : 1;
      k_gather_xyz_packed<<<dim3((unsigned) xyz_gx, (unsigned) nf, (unsigned) nparts), XYZ_THREADS, 0, s>>>(
          ctx->d_in.p, ctx->d_pt_off.p, ctx->d_counts.p, nf, ctx->d_out_idx.p, b.d_pg_off.p, b.d_png_off.p, first, b.d_pgxyz.p, b.d_pngxyz.p);
      ++ctx->launches;
    }
    if (b.packed_rec) {   // the records the runs read, as k_gather_record_parts reads them
      const int first = b.packed_rec == PWPP_PART_NONGROUND ? 1 : 0, nparts = b.packed_rec == 3 ? 2 : 1;
      k_gather_record_packed<<<dim3((unsigned) rec_gx, (unsigned) nf, (unsigned) nparts), REC_THREADS, 0, s>>>(
          recs, ctx->d_pt_off.p, ctx->d_counts.p, nf, ctx->d_out_idx.p, b.d_pg_off.p, b.d_png_off.p, first, b.d_prec_g.p, b.d_prec_ng.p);
      ++ctx->launches;
    }
    CU_TRY(cudaGetLastError());
  }
  return PWPP_OK;
}

// A laddered run of bound call b into the graph that s is capturing: the table kernel, k_ladder_select, and a SWITCH node whose
// body i is a child graph node holding a copy of L.bodies[i]. Conditional bodies may hold child graphs but no event nodes, which
// is why the bodies (whose fit kernels fork to the side streams) are captured beforehand, outside any caller's capture.
static int enqueue_ladder(pwpp_ctx* ctx, pwpp_ctx::Bound& b, const BoundLadder& L, cudaStream_t s) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  cudaGraph_t g = nullptr;
  CU_TRY(cudaStreamGetCaptureInfo_v3(s, &st, nullptr, &g));
  if (st != cudaStreamCaptureStatusActive) return fail(PWPP_ERR_CUDA, "the stream's capture was invalidated");
  cudaGraphConditionalHandle h;
  CU_TRY(cudaGraphConditionalHandleCreate(&h, g, 0, cudaGraphCondAssignDefault));
  int rc = enqueue_bound_table(ctx, b, s);
  if (rc) return rc;
  k_ladder_select<<<1, LS_THREADS, 0, s>>>(b.nf, b.d_bstatus.p, L.widths, b.d_width.p, h);
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  const cudaGraphNode_t* deps = nullptr;
  const cudaGraphEdgeData* edges = nullptr;
  size_t ndeps = 0;
  CU_TRY(cudaStreamGetCaptureInfo_v3(s, &st, nullptr, &g, &deps, &edges, &ndeps));
  cudaGraphNodeParams p = {};
  p.type = cudaGraphNodeTypeConditional;
  p.conditional.handle = h;
  p.conditional.type = cudaGraphCondTypeSwitch;
  p.conditional.size = (unsigned) L.widths.n;
  cudaGraphNode_t node;
  CU_TRY(cudaGraphAddNode_v2(&node, g, deps, edges, ndeps, &p));
  for (int i = 0; i < L.widths.n; ++i) {
    cudaGraphNode_t child;
    CU_TRY(cudaGraphAddChildGraphNode(&child, p.conditional.phGraph_out[i], nullptr, 0, L.bodies[i]));
  }
  CU_TRY(cudaStreamUpdateCaptureDependencies_v2(s, &node, nullptr, 1, cudaStreamSetCaptureDependencies));
  ctx->launches += L.body_launches;
  return PWPP_OK;
}

// One table launch, then the body: one unpack launch (capacities with points), every run through launch_range_impl with grids
// sized for its capacities, and the gathers. Never through launch_range: its own capture would nest inside a caller's. With a
// width ladder the body is the SWITCH node of enqueue_ladder: captured into the caller's graph when s is capturing, otherwise
// launched as the ladder's own executable graph.
int pwpp_run_bound_call(pwpp_ctx* ctx, void* cuda_stream) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->bound[ctx->sel].on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  int rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  const int k = ctx->sel;   // a graph captured from here holds this call, whatever is selected later
  pwpp_ctx::Bound& b = ctx->bound[k];
  describe_bound(ctx, b);
  b.ran = true;
  if (b.ladder) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    CU_TRY(cudaStreamIsCapturing(s, &st));
    if (st != cudaStreamCaptureStatusNone) {
      rc = enqueue_ladder(ctx, b, *b.ladder, s);
      if (rc) return rc;
    } else {
      CU_TRY(cudaGraphLaunch(b.ladder->exec, s));
      ctx->launches += b.ladder->launches;
    }
  } else {
    rc = enqueue_bound_table(ctx, b, s);
    if (rc) return rc;
    rc = enqueue_bound_body(ctx, b, s, b.nf);
    if (rc) return rc;
  }
  make_bound_last(ctx, k, s);
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

int pwpp_bound_call_results(pwpp_ctx* ctx, const int32_t** d_indices, const int64_t** d_offsets, const int32_t** d_num_ground,
                            const int32_t** d_status) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->bound[ctx->sel].on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  make_bound_last(ctx, ctx->sel, ctx->last_stream ? ctx->last_stream : ctx->stream);
  if (d_indices) *d_indices = ctx->d_out_idx.p;
  if (d_offsets) *d_offsets = reinterpret_cast<const int64_t*>(ctx->d_pt_off.p);
  if (d_num_ground) *d_num_ground = ctx->d_counts.p;
  if (d_status) *d_status = ctx->bound[ctx->sel].d_bstatus.p;
  return PWPP_OK;
}

int pwpp_bound_call_slots(pwpp_ctx* ctx, const int32_t** d_slots_read) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->bound[ctx->sel].on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call_rings)");
  if (!ctx->bound[ctx->sel].d_slots) return fail(PWPP_ERR_INVALID_ARG, "the bound call has no rings (pwpp_bind_call_rings)");
  if (d_slots_read) *d_slots_read = ctx->bound[ctx->sel].d_bslot.p;
  return PWPP_OK;
}

// With a stream table every frame of run r gets scratch slot num_streams + (f - runs[r]) as with actions, and dep[f] = (r > 0):
// the table kernel resets the RESET frames of run 0, k_bound_reset those of every later run (the host no longer knows which
// streams repeat). The tables are built in buffers of their own and moved into the bound call only when all of them exist.
int pwpp_bind_stream_table(pwpp_ctx* ctx, const int32_t* d_streams) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (!d_streams) return fail(PWPP_ERR_INVALID_ARG, "d_streams is NULL");
  int rc = check_no_ladder(b, "the stream table");
  if (rc) return rc;
  if (b.d_streams) return fail(PWPP_ERR_INVALID_ARG, "a stream table is already enabled for the bound call");
  if (b.ran)
    return fail(PWPP_ERR_INVALID_ARG, "the bound call has run or been captured: enable its stream table before its first run (the state buffers may grow)");
  rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = b.nf, nruns = (int) b.runs.size() - 1, ns = ctx->num_streams;
  std::vector<int> scratch(nf), dep(nf);
  int slots = 0;   // the longest run
  for (int r = 0; r < nruns; ++r) {
    slots = std::max(slots, b.runs[r + 1] - b.runs[r]);
    for (int f = b.runs[r]; f < b.runs[r + 1]; ++f) {
      scratch[f] = ns + (f - b.runs[r]);
      dep[f] = r > 0;
    }
  }
  if ((rc = check_growth(ctx, slots))) return rc;
  // the state buffers may move: whatever the ctx enqueued before has finished with them
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  if (slots > ctx->scratch_slots) {
    const size_t n = (size_t) ns + slots;
    CU_TRY(ctx->d_states.grow_keep(n));
    CU_TRY(ctx->d_hist.grow_keep(n * 2 * 4 * ctx->hist_stride));
    ctx->scratch_slots = slots;
  }
  if (!b.d_actions) {   // (with actions the bind filled them) a scratch slot starts as a constructor state, as in bind_call_impl
    StreamState s0;
    CU_TRY(cudaMemcpy(&s0, ctx->d_states_init.p, sizeof(StreamState), cudaMemcpyDeviceToHost));
    const std::vector<StreamState> fill(slots, s0);
    CU_TRY(cudaMemcpy(ctx->d_states.p + ns, fill.data(), (size_t) slots * sizeof(StreamState), cudaMemcpyHostToDevice));
  }
  DevBuf<int, false> read, claim, set_of, runs, sc, dp;
  CU_TRY(read.reserve(nf));
  CU_TRY(claim.reserve(ns));
  CU_TRY(set_of.reserve(ns));
  CU_TRY(runs.reserve(nruns + 1));
  CU_TRY(sc.reserve(nf));
  CU_TRY(dp.reserve(nf));
  CU_TRY(cudaMemset(read.p, 0xff, (size_t) nf * sizeof(int)));   // -1: no run yet
  CU_TRY(cudaMemset(claim.p, 0xff, (size_t) ns * sizeof(int)));
  CU_TRY(cudaMemcpy(set_of.p, ctx->stream_set.data(), (size_t) ns * sizeof(int), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(runs.p, b.runs.data(), (size_t) (nruns + 1) * sizeof(int), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(sc.p, scratch.data(), (size_t) nf * sizeof(int), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(dp.p, dep.data(), (size_t) nf * sizeof(int), cudaMemcpyHostToDevice));
  CU_TRY(cudaDeviceSynchronize());
  b.d_bread = std::move(read);
  b.d_bclaim = std::move(claim);
  b.d_bset_of = std::move(set_of);
  b.d_bruns = std::move(runs);
  b.d_bscratch = std::move(sc);
  if (b.d_actions) b.d_bdep = std::move(dp);
  b.d_streams = d_streams;
  return PWPP_OK;
}

int pwpp_bound_call_streams(pwpp_ctx* ctx, const int32_t** d_streams_read) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->bound[ctx->sel].on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (!ctx->bound[ctx->sel].d_streams) return fail(PWPP_ERR_INVALID_ARG, "the bound call has no stream table (pwpp_bind_stream_table)");
  if (d_streams_read) *d_streams_read = ctx->bound[ctx->sel].d_bread.p;
  return PWPP_OK;
}

int pwpp_unbind_call(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->bound[ctx->sel].on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound");
  int rc = bind_device(ctx);
  if (rc) return rc;
  ctx->bound[ctx->sel] = pwpp_ctx::Bound();   // releases the bound call's buffers; no shared buffer moves
  return PWPP_OK;
}

// One plain graph per width, each captured on the ctx's own stream outside any caller's capture (the body forks to the side
// streams), then the whole run (enqueue_ladder) captured once more into the executable graph of uncaptured runs. The host
// description and the launch counter are the ctx's again afterwards: the enable is no run.
int pwpp_bind_width_ladder(pwpp_ctx* ctx, int nwidths, const int32_t* widths) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (b.ladder) return fail(PWPP_ERR_INVALID_ARG, "a width ladder is already enabled for the bound call");
  if (!b.d_actions && !b.d_streams)
    return fail(PWPP_ERR_INVALID_ARG, "the bound call has neither actions nor a stream table: every position runs, so the ladder would always pick the full width");
  if (!widths) return fail(PWPP_ERR_INVALID_ARG, "widths is NULL");
  if (nwidths < 1 || nwidths > PWPP_MAX_LADDER_WIDTHS - 1)
    return fail(PWPP_ERR_INVALID_ARG, "nwidths must be in [1, " + std::to_string(PWPP_MAX_LADDER_WIDTHS - 1) + "] (nframes is the implicit last width)");
  auto L = std::make_unique<BoundLadder>();
  for (int i = 0; i < nwidths; ++i) {
    if (widths[i] < 1 || widths[i] >= b.nf || (i > 0 && widths[i] <= widths[i - 1]))
      return fail(PWPP_ERR_INVALID_ARG, "widths[" + std::to_string(i) + "] = " + std::to_string(widths[i]) +
                                            ": widths must be strictly increasing and in [1, nframes = " + std::to_string(b.nf) + ")");
    L->widths.w[i] = widths[i];
  }
  L->widths.w[nwidths] = b.nf;
  L->widths.n = nwidths + 1;
  int rc = bind_device(ctx);
  if (rc) return rc;
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  const int saved_nframes = ctx->last_nframes;
  const std::vector<int> saved_runs = ctx->runs, saved_set = ctx->frame_set, saved_chunk = ctx->chunk_off;
  const std::vector<long long> saved_pt = ctx->pt_off;
  const bool saved_dev = ctx->sets_on_device;
  const float4* saved_pts = ctx->last_pts;
  const cudaStream_t saved_stream = ctx->last_stream;
  const long long saved_launches = ctx->launches;
  // a failed capture ends it here (cudaStreamEndCapture) and leaves its partial graph to L
  auto capture = [&](cudaGraph_t* out, auto&& enqueue) -> int {
    cudaStream_t s = ctx->stream;
    CU_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue(s);
    const cudaError_t e = cudaStreamEndCapture(s, out);
    if (rc) return rc;
    CU_TRY(e);
    return PWPP_OK;
  };
  auto build = [&]() -> int {
    describe_bound(ctx, b);
    for (int i = 0; i < L->widths.n; ++i) {
      const long long l0 = ctx->launches;
      cudaGraph_t g = nullptr;
      const int rc = capture(&g, [&](cudaStream_t s) { return enqueue_bound_body(ctx, b, s, L->widths.w[i]); });
      if (g) L->bodies.push_back(g);
      if (rc) return rc;
      L->body_launches = ctx->launches - l0;   // the last one, nframes wide, stays
    }
    const long long l0 = ctx->launches;
    cudaGraph_t g = nullptr;
    int rc = capture(&g, [&](cudaStream_t s) { return enqueue_ladder(ctx, b, *L, s); });
    if (rc == PWPP_OK) {
      const cudaError_t e = cudaGraphInstantiate(&L->exec, g, 0);
      if (e != cudaSuccess) {
        L->exec = nullptr;
        rc = fail(PWPP_ERR_CUDA, std::string("instantiating the width ladder's graph: ") + cudaGetErrorString(e));
      }
    }
    if (g) cudaGraphDestroy(g);
    if (rc) return rc;
    L->launches = ctx->launches - l0;
    CU_TRY(cudaMemset(b.d_width.p, 0, sizeof(int)));
    CU_TRY(cudaDeviceSynchronize());
    return PWPP_OK;
  };
  rc = build();
  ctx->last_nframes = saved_nframes;
  ctx->runs = saved_runs;
  ctx->frame_set = saved_set;
  ctx->chunk_off = saved_chunk;
  ctx->pt_off = saved_pt;
  ctx->sets_on_device = saved_dev;
  ctx->last_pts = saved_pts;
  ctx->last_stream = saved_stream;
  ctx->launches = saved_launches;
  if (rc) {
    cudaGetLastError();
    return rc;
  }
  b.ladder = std::move(L);
  b.ran = true;   // its graphs hold the shared buffers: no later bind may grow them
  return PWPP_OK;
}

int pwpp_bound_call_width(pwpp_ctx* ctx, const int32_t** d_width) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->bound[ctx->sel].on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (d_width) *d_width = ctx->bound[ctx->sel].d_width.p;
  return PWPP_OK;
}

int pwpp_select_bound_call(pwpp_ctx* ctx, int k) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (k < 0 || k >= PWPP_MAX_BOUND_CALLS)
    return fail(PWPP_ERR_INVALID_ARG, "bound call " + std::to_string(k) + " is outside [0, " + std::to_string(PWPP_MAX_BOUND_CALLS) + ")");
  ctx->sel = k;
  return PWPP_OK;
}

int pwpp_selected_bound_call(const pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  return ctx->sel;
}

int pwpp_bind_record_results(pwpp_ctx* ctx, int parts) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (parts < 1 || parts > 3) return fail(PWPP_ERR_INVALID_ARG, "parts must be PWPP_PART_GROUND, PWPP_PART_NONGROUND or both");
  int rc = check_no_ladder(b, "record results");
  if (rc) return rc;
  if (b.rec_parts) return fail(PWPP_ERR_INVALID_ARG, "record results are already enabled for the bound call");
  rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = b.nf;
  std::vector<long long> off(nf + 1);   // the direct call's region layout with n = max_n
  rec_out_offsets(b.cap_pt_off.data(), b.recs.data(), nf, off.data());
  const size_t bytes = (size_t) std::max<long long>(off[nf], 16);
  if (parts & PWPP_PART_GROUND) CU_TRY(b.d_bground.reserve(bytes));
  if (parts & PWPP_PART_NONGROUND) CU_TRY(b.d_bnonground.reserve(bytes));
  CU_TRY(b.d_bpart_off.reserve(nf + 1));
  CU_TRY(b.d_rec_counts.reserve(2 * (size_t) nf));
  CU_TRY(cudaMemcpy(b.d_bpart_off.p, off.data(), (size_t) (nf + 1) * sizeof(long long), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemset(b.d_rec_counts.p, 0, 2 * (size_t) nf * sizeof(int)));
  CU_TRY(cudaDeviceSynchronize());
  b.rec_part_off = std::move(off);
  b.rec_parts = parts;
  return PWPP_OK;
}

int pwpp_bound_record_results(pwpp_ctx* ctx, const void** d_ground, const void** d_nonground, const int64_t** h_offsets,
                              const int32_t** d_counts) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (!b.rec_parts) return fail(PWPP_ERR_INVALID_ARG, "record results are not enabled for the bound call (pwpp_bind_record_results)");
  if (d_ground) *d_ground = (b.rec_parts & PWPP_PART_GROUND) ? b.d_bground.p : nullptr;
  if (d_nonground) *d_nonground = (b.rec_parts & PWPP_PART_NONGROUND) ? b.d_bnonground.p : nullptr;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(b.rec_part_off.data());
  if (d_counts) *d_counts = b.d_rec_counts.p;
  return PWPP_OK;
}

int pwpp_bind_getter_results(pwpp_ctx* ctx, int what) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (what < 1 || what > 7) return fail(PWPP_ERR_INVALID_ARG, "what must be a non-empty set of PWPP_GETTER_GROUND_XYZ, PWPP_GETTER_NONGROUND_XYZ and PWPP_GETTER_STATE");
  int rc = check_no_ladder(b, "getter results");
  if (rc) return rc;
  if (b.getters) return fail(PWPP_ERR_INVALID_ARG, "getter results are already enabled for the bound call");
  rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = b.nf;
  const size_t rows = (size_t) std::max<long long>(b.cap_pt_off[nf], 1);
  if (what & PWPP_GETTER_GROUND_XYZ) CU_TRY(b.d_bgxyz.reserve(3 * rows));
  if (what & PWPP_GETTER_NONGROUND_XYZ) CU_TRY(b.d_bngxyz.reserve(3 * rows));
  if (what & (PWPP_GETTER_GROUND_XYZ | PWPP_GETTER_NONGROUND_XYZ)) {
    CU_TRY(b.d_bxyz_off.reserve(nf + 1));
    CU_TRY(b.d_xyz_counts.reserve(2 * (size_t) nf));
    CU_TRY(cudaMemcpy(b.d_bxyz_off.p, b.cap_pt_off.data(), (size_t) (nf + 1) * sizeof(long long), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemset(b.d_xyz_counts.p, 0, 2 * (size_t) nf * sizeof(int)));
  }
  if (what & PWPP_GETTER_STATE) {
    CU_TRY(b.d_bstates.reserve(nf));
    CU_TRY(cudaMemset(b.d_bstates.p, 0, (size_t) nf * sizeof(pwpp_state)));
  }
  CU_TRY(cudaDeviceSynchronize());
  b.getters = what;
  return PWPP_OK;
}

// The ground and non-ground offsets that packed xyz and packed records share (k_bound_xyz_offsets writes both at every run):
// reserved and zeroed by whichever of the two is enabled first.
static int reserve_packed_offsets(pwpp_ctx::Bound& b) {
  if (b.packed_xyz || b.packed_rec) return PWPP_OK;
  CU_TRY(b.d_pg_off.reserve(b.nf + 1));
  CU_TRY(b.d_png_off.reserve(b.nf + 1));
  CU_TRY(cudaMemset(b.d_pg_off.p, 0, (size_t) (b.nf + 1) * sizeof(long long)));
  CU_TRY(cudaMemset(b.d_png_off.p, 0, (size_t) (b.nf + 1) * sizeof(long long)));
  return PWPP_OK;
}

int pwpp_bind_packed_xyz(pwpp_ctx* ctx, int parts) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (parts < 1 || parts > 3) return fail(PWPP_ERR_INVALID_ARG, "parts must be PWPP_PART_GROUND, PWPP_PART_NONGROUND or both");
  int rc = check_no_ladder(b, "packed xyz");
  if (rc) return rc;
  if (b.packed_xyz) return fail(PWPP_ERR_INVALID_ARG, "packed xyz is already enabled for the bound call");
  rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = b.nf;
  const size_t rows = (size_t) std::max<long long>(b.cap_pt_off[nf], 1);
  if (parts & PWPP_PART_GROUND) CU_TRY(b.d_pgxyz.reserve(3 * rows));
  if (parts & PWPP_PART_NONGROUND) CU_TRY(b.d_pngxyz.reserve(3 * rows));
  if ((rc = reserve_packed_offsets(b))) return rc;
  CU_TRY(cudaDeviceSynchronize());
  b.packed_xyz = parts;
  return PWPP_OK;
}

int pwpp_bind_packed_records(pwpp_ctx* ctx, int parts) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (parts < 1 || parts > 3) return fail(PWPP_ERR_INVALID_ARG, "parts must be PWPP_PART_GROUND, PWPP_PART_NONGROUND or both");
  int rc = check_no_ladder(b, "packed records");
  if (rc) return rc;
  if (b.packed_rec) return fail(PWPP_ERR_INVALID_ARG, "packed records are already enabled for the bound call");
  const int nf = b.nf;
  for (int f = 1; f < nf; ++f)   // one step for the whole buffer: each part is one (rows, point_step) byte array
    if (b.recs[f].step != b.recs[0].step)
      return fail(PWPP_ERR_UNSUPPORTED, "frame " + std::to_string(f) + " has point_step " + std::to_string(b.recs[f].step) + ", frame 0 has " +
                                            std::to_string(b.recs[0].step) + ": packed records need one point_step (pwpp_bind_record_results does not)");
  rc = bind_device(ctx);
  if (rc) return rc;
  const size_t bytes = (size_t) std::max<long long>(b.cap_pt_off[nf], 1) * (size_t) b.recs[0].step;
  if (parts & PWPP_PART_GROUND) CU_TRY(b.d_prec_g.reserve(bytes));
  if (parts & PWPP_PART_NONGROUND) CU_TRY(b.d_prec_ng.reserve(bytes));
  if ((rc = reserve_packed_offsets(b))) return rc;
  CU_TRY(cudaDeviceSynchronize());
  b.packed_rec = parts;
  return PWPP_OK;
}

int pwpp_bound_packed_records(pwpp_ctx* ctx, const void** d_ground, const void** d_nonground, const int64_t** d_ground_off,
                              const int64_t** d_nonground_off, int32_t* point_step) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (!b.packed_rec) return fail(PWPP_ERR_INVALID_ARG, "packed records are not enabled for the bound call (pwpp_bind_packed_records)");
  const bool g = b.packed_rec & PWPP_PART_GROUND, n = b.packed_rec & PWPP_PART_NONGROUND;
  if (d_ground) *d_ground = g ? b.d_prec_g.p : nullptr;
  if (d_nonground) *d_nonground = n ? b.d_prec_ng.p : nullptr;
  if (d_ground_off) *d_ground_off = g ? reinterpret_cast<const int64_t*>(b.d_pg_off.p) : nullptr;
  if (d_nonground_off) *d_nonground_off = n ? reinterpret_cast<const int64_t*>(b.d_png_off.p) : nullptr;
  if (point_step) *point_step = b.recs[0].step;
  return PWPP_OK;
}

int pwpp_bound_packed_xyz(pwpp_ctx* ctx, const float** d_ground, const float** d_nonground, const int64_t** d_ground_off,
                          const int64_t** d_nonground_off) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  if (!b.packed_xyz) return fail(PWPP_ERR_INVALID_ARG, "packed xyz is not enabled for the bound call (pwpp_bind_packed_xyz)");
  const bool g = b.packed_xyz & PWPP_PART_GROUND, n = b.packed_xyz & PWPP_PART_NONGROUND;
  if (d_ground) *d_ground = g ? b.d_pgxyz.p : nullptr;
  if (d_nonground) *d_nonground = n ? b.d_pngxyz.p : nullptr;
  if (d_ground_off) *d_ground_off = g ? reinterpret_cast<const int64_t*>(b.d_pg_off.p) : nullptr;
  if (d_nonground_off) *d_nonground_off = n ? reinterpret_cast<const int64_t*>(b.d_png_off.p) : nullptr;
  return PWPP_OK;
}

int pwpp_bound_getter_results(pwpp_ctx* ctx, pwpp_bound_getters* out) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  const pwpp_ctx::Bound& b = ctx->bound[ctx->sel];
  if (!b.on) return fail(PWPP_ERR_INVALID_ARG, "no call is bound (pwpp_bind_call)");
  *out = pwpp_bound_getters{};
  out->ground_xyz = (b.getters & PWPP_GETTER_GROUND_XYZ) ? b.d_bgxyz.p : nullptr;
  out->nonground_xyz = (b.getters & PWPP_GETTER_NONGROUND_XYZ) ? b.d_bngxyz.p : nullptr;
  out->h_row_off = reinterpret_cast<const int64_t*>(b.cap_pt_off.data());
  out->xyz_counts = (b.getters & 3) ? b.d_xyz_counts.p : nullptr;
  out->centers = ctx->d_centers.p;
  out->normals = ctx->d_normals.p;
  out->num_patches = ctx->d_counts.p + b.nf;   // row 1 of the count rows of the bound call
  out->patch_row_stride = ctx->gs.nbs;
  out->states = (b.getters & PWPP_GETTER_STATE) ? b.d_bstates.p : nullptr;
  return PWPP_OK;
}

// Record results of the last call: the first request gathers every frame's records into d_rec_out on the call's stream (one
// launch, none when the call had no points), and no later request of the same call gathers again. The host blocks only where
// a buffer is first reserved or grows, and on the previous request's offset-table upload (include/pwpp.h).
static int gather_records(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (ctx->last_nframes <= 0) return fail(PWPP_ERR_INVALID_ARG, "no estimate call yet");
  if (ctx->last_call >= 0)
    return fail(PWPP_ERR_INVALID_ARG, "record results are not available for a bound call (pwpp_run_bound_call): their gather needs host offsets (pwpp_bind_record_results gives a bound call its own)");
  if (ctx->last_recs.empty()) return fail(PWPP_ERR_INVALID_ARG, "the last estimate call did not take records (pwpp_estimate_host_records / pwpp_estimate_device_records)");
  if (ctx->rec_gathered) return PWPP_OK;
  int rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = ctx->last_nframes;
  cudaStream_t s = ctx->last_stream;
  ctx->rec_off.assign(nf + 1, 0);
  rec_out_offsets(ctx->pt_off.data(), ctx->last_recs.data(), nf, ctx->rec_off.data());
  CU_TRY(ctx->d_rec_out.reserve((size_t) std::max<long long>(ctx->rec_off[nf], 16)));
  CU_TRY(ctx->d_rec_off.reserve(nf + 1));
  if (ctx->ev_rec_off) CU_TRY(cudaEventSynchronize(ctx->ev_rec_off));   // the previous gather's upload has read the staging
  else CU_TRY(cudaEventCreateWithFlags(&ctx->ev_rec_off, cudaEventDisableTiming));
  CU_TRY(ctx->h_rec_off.reserve(nf + 1));
  std::memcpy(ctx->h_rec_off.p, ctx->rec_off.data(), (size_t) (nf + 1) * sizeof(long long));
  CU_TRY(cudaMemcpyAsync(ctx->d_rec_off.p, ctx->h_rec_off.p, (size_t) (nf + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaEventRecord(ctx->ev_rec_off, s));
  if (ctx->last_total > 0) {
    const long long gx = rec_grid_x(ctx->pt_off.data(), ctx->last_recs.data(), nf);
    k_gather_records<<<dim3((unsigned) gx, (unsigned) nf), REC_THREADS, 0, s>>>(ctx->d_rec.p, ctx->d_pt_off.p, ctx->d_rec_off.p, ctx->d_counts.p + 2 * nf,
                                                                               ctx->d_out_idx.p, ctx->d_rec_out.p);
    ++ctx->launches;
    CU_TRY(cudaGetLastError());
  }
  ctx->rec_gathered = true;
  return PWPP_OK;
}

// The gathered records in the page-locked host view (one D2H per call), and the counts.
static int fetch_records(pwpp_ctx* ctx) {
  int rc = gather_records(ctx);
  if (rc) return rc;
  rc = fetch_counts(ctx);
  if (rc) return rc;
  if (ctx->rec_fetched) return PWPP_OK;
  const long long bytes = ctx->rec_off[ctx->last_nframes];
  CU_TRY(ctx->h_rec_out.reserve((size_t) std::max<long long>(bytes, 16)));
  if (bytes > 0) CU_TRY(cudaMemcpyAsync(ctx->h_rec_out.p, ctx->d_rec_out.p, (size_t) bytes, cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->rec_fetched = true;
  return PWPP_OK;
}

int pwpp_device_record_results(pwpp_ctx* ctx, const void** d_records, const int64_t** h_offsets) {
  const int rc = gather_records(ctx);
  if (rc) return rc;
  if (d_records) *d_records = ctx->d_rec_out.p;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(ctx->rec_off.data());
  return PWPP_OK;
}
int pwpp_host_record_results(pwpp_ctx* ctx, const void** h_records, const int64_t** h_offsets) {
  const int rc = fetch_records(ctx);
  if (rc) return rc;
  if (h_records) *h_records = ctx->h_rec_out.p;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(ctx->rec_off.data());
  return PWPP_OK;
}
static int copy_records(pwpp_ctx* ctx, int f, void* dst, bool ground) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_records(ctx);
  if (rc) return rc;
  const long long step = ctx->last_recs[f].step;
  const FrameList L = frame_list(ctx, f, ground);
  if (L.count > 0) std::memcpy(dst, ctx->h_rec_out.p + ctx->rec_off[f] + L.start * step, (size_t) (L.count * step));
  return PWPP_OK;
}
int pwpp_copy_ground_records(pwpp_ctx* ctx, int f, void* dst) { return copy_records(ctx, f, dst, true); }
int pwpp_copy_nonground_records(pwpp_ctx* ctx, int f, void* dst) { return copy_records(ctx, f, dst, false); }

int pwpp_device_synchronize(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaDeviceSynchronize());
  return PWPP_OK;
}

int pwpp_synchronize(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaStreamSynchronize(ctx->last_stream ? ctx->last_stream : ctx->stream));
  return PWPP_OK;
}

int64_t pwpp_num_ground(pwpp_ctx* ctx, int f) {
  if (check_frame(ctx, f) || fetch_counts(ctx)) return -1;
  return ctx->h_counts.p[f];
}
int64_t pwpp_num_nonground(pwpp_ctx* ctx, int f) {
  if (check_frame(ctx, f) || fetch_counts(ctx)) return -1;
  return frame_list(ctx, f, false).count;
}
static int copy_indices(pwpp_ctx* ctx, int f, int32_t* dst, bool ground) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_indices(ctx);
  if (rc) return rc;
  const FrameList L = frame_list(ctx, f, ground);
  if (L.count > 0) std::memcpy(dst, ctx->h_out_idx.p + ctx->pt_off[f] + L.start, (size_t) L.count * sizeof(int32_t));
  return PWPP_OK;
}
int pwpp_copy_ground_indices(pwpp_ctx* ctx, int f, int32_t* dst) { return copy_indices(ctx, f, dst, true); }
int pwpp_copy_nonground_indices(pwpp_ctx* ctx, int f, int32_t* dst) { return copy_indices(ctx, f, dst, false); }

static int copy_xyz(pwpp_ctx* ctx, int f, float* dst, bool ground) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_counts(ctx);
  if (rc) return rc;
  const FrameList L = frame_list(ctx, f, ground);
  const int cnt = L.count;
  if (cnt <= 0) return PWPP_OK;
  CU_TRY(ctx->d_xyz.reserve((size_t) cnt * 3));
  const int* idx = ctx->d_out_idx.p + ctx->pt_off[f] + L.start;
  k_gather_xyz<<<(cnt + 255) / 256, 256, 0, ctx->last_stream>>>(ctx->last_pts + ctx->pt_off[f], idx, cnt, ctx->d_xyz.p);
  CU_TRY(cudaGetLastError());
  CU_TRY(cudaMemcpyAsync(dst, ctx->d_xyz.p, (size_t) cnt * 3 * sizeof(float), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  return PWPP_OK;
}
int pwpp_copy_ground_xyz(pwpp_ctx* ctx, int f, float* dst) { return copy_xyz(ctx, f, dst, true); }
int pwpp_copy_nonground_xyz(pwpp_ctx* ctx, int f, float* dst) { return copy_xyz(ctx, f, dst, false); }

int pwpp_num_patches(pwpp_ctx* ctx, int f) {
  if (check_frame(ctx, f) || fetch_counts(ctx)) return -1;
  return count_of(ctx, 1, f);
}
int pwpp_copy_centers(pwpp_ctx* ctx, int f, float* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_patches(ctx);
  if (rc) return rc;
  const int k = count_of(ctx, 1, f);
  if (k > 0) std::memcpy(dst, ctx->h_centers.p + (size_t) f * ctx->gs.nbs * 3, (size_t) k * 3 * sizeof(float));
  return PWPP_OK;
}
int pwpp_copy_normals(pwpp_ctx* ctx, int f, float* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_patches(ctx);
  if (rc) return rc;
  const int k = count_of(ctx, 1, f);
  if (k > 0) std::memcpy(dst, ctx->h_normals.p + (size_t) f * ctx->gs.nbs * 3, (size_t) k * 3 * sizeof(float));
  return PWPP_OK;
}

int pwpp_get_state(pwpp_ctx* ctx, int f, pwpp_state* out) {
  if (!ctx || !out || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  int rc = bind_device(ctx);
  if (rc) return rc;
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  StreamState s;
  CU_TRY(cudaMemcpy(&s, ctx->d_states.p + f, sizeof(s), cudaMemcpyDeviceToHost));
  out->sensor_height = s.sensor_height;
  for (int i = 0; i < 4; ++i) {
    out->elevation_thr[i] = s.elevation_thr[i]; out->flatness_thr[i] = s.flatness_thr[i];
    out->n_elevation[i] = s.n_elev[i]; out->n_flatness[i] = s.n_flat[i];
  }
  return PWPP_OK;
}
double pwpp_height(pwpp_ctx* ctx, int f) {
  pwpp_state s;
  if (pwpp_get_state(ctx, f, &s)) return NAN;
  return s.sensor_height;
}
double pwpp_time_us(pwpp_ctx* ctx) { return ctx ? ctx->last_time_us : NAN; }

int pwpp_call_times_us(pwpp_ctx* ctx, float out[4]) {
  if (!ctx || !out) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (!ctx->call_times_valid) return fail(PWPP_ERR_INVALID_ARG, "no single-chunk pwpp_estimate_host call to report on");
  int rc = bind_device(ctx);
  if (rc) return rc;
  float ms[4];
  CU_TRY(cudaEventElapsedTime(&ms[0], ctx->ev_begin, ctx->ev0));
  CU_TRY(cudaEventElapsedTime(&ms[1], ctx->ev0, ctx->ev1));
  CU_TRY(cudaEventElapsedTime(&ms[2], ctx->ev1, ctx->ev_end));
  CU_TRY(cudaEventElapsedTime(&ms[3], ctx->ev_begin, ctx->ev_end));
  for (int i = 0; i < 4; ++i) out[i] = ms[i] * 1000.f;
  return PWPP_OK;
}

int pwpp_copy_history(pwpp_ctx* ctx, int f, int ring, int which, double* dst) {
  if (!ctx || !dst || f < 0 || f >= ctx->num_streams || ring < 0 || ring > 3 || which < 0 || which > 1) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  pwpp_state s;
  int rc = pwpp_get_state(ctx, f, &s);
  if (rc) return rc;
  const int n = which ? s.n_flatness[ring] : s.n_elevation[ring];
  if (n > 0) CU_TRY(cudaMemcpy(dst, ctx->d_hist.p + (((size_t) f * 2 + which) * 4 + ring) * ctx->hist_stride, (size_t) n * sizeof(double), cudaMemcpyDeviceToHost));
  return PWPP_OK;
}

// a stream's blob: header, state, then its eight history rows of its own set's capacity (the layout of a one-set context)
static size_t blob_size_of_cap(int hcap) { return state_blob_bytes(hcap); }
size_t pwpp_stream_state_blob_size(const pwpp_ctx* ctx, int s) {
  if (!ctx || s < 0 || s >= ctx->num_streams) return 0;
  return blob_size_of_cap(ctx->set_hcap[ctx->stream_set[s]]);
}
size_t pwpp_state_blob_size(const pwpp_ctx* ctx) { return ctx ? blob_size_of_cap(ctx->hist_stride) : 0; }
int pwpp_export_state(pwpp_ctx* ctx, int f, void* blob) {
  if (!ctx || !blob || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  int rc = bind_device(ctx);
  if (rc) return rc;
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  char* b = static_cast<char*>(blob);
  const int hcap = ctx->set_hcap[ctx->stream_set[f]];
  const StateBlobHeader h{STATE_BLOB_MAGIC, (uint32_t) PWPP_ABI_VERSION, hcap, (int32_t) sizeof(StreamState)};
  std::memcpy(b, &h, sizeof h);
  CU_TRY(cudaMemcpy(b + sizeof h, ctx->d_states.p + f, sizeof(StreamState), cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemcpy2D(b + sizeof h + sizeof(StreamState), (size_t) hcap * sizeof(double), ctx->d_hist.p + (size_t) f * 2 * 4 * ctx->hist_stride,
                      (size_t) ctx->hist_stride * sizeof(double), (size_t) hcap * sizeof(double), 2 * 4, cudaMemcpyDeviceToHost));
  return PWPP_OK;
}
int pwpp_import_state(pwpp_ctx* ctx, int f, const void* blob, size_t bytes) {
  if (!ctx || !blob || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  if (bytes != pwpp_stream_state_blob_size(ctx, f)) return fail(PWPP_ERR_INVALID_ARG, "state blob has the wrong size for this context (different storage parameters?)");
  const int hcap = ctx->set_hcap[ctx->stream_set[f]];
  const char* b = static_cast<const char*>(blob);
  StateBlobHeader h;
  std::memcpy(&h, b, sizeof h);
  if (h.magic != STATE_BLOB_MAGIC || h.version != (uint32_t) PWPP_ABI_VERSION || h.hcap != hcap || h.state_bytes != (int32_t) sizeof(StreamState))
    return fail(PWPP_ERR_INVALID_ARG, "not a state blob of this library version / parameter set");
  int rc = bind_device(ctx);
  if (rc) return rc;
  // after everything already enqueued (a synchronous copy from pageable memory: the blob may be freed on return)
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  CU_TRY(cudaMemcpy(ctx->d_states.p + f, b + sizeof h, sizeof(StreamState), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy2D(ctx->d_hist.p + (size_t) f * 2 * 4 * ctx->hist_stride, (size_t) ctx->hist_stride * sizeof(double), b + sizeof h + sizeof(StreamState),
                      (size_t) hcap * sizeof(double), (size_t) hcap * sizeof(double), 2 * 4, cudaMemcpyHostToDevice));
  return PWPP_OK;
}

// The host checks of pwpp_export_states_device / pwpp_import_states_device; *run = false when there is nothing to launch.
static int check_state_list(const pwpp_ctx* ctx, int n, const int32_t* d_streams, const void* d_blobs, int64_t blob_stride, bool* run) {
  *run = false;
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (n < 0 || n > 65535) return fail(PWPP_ERR_INVALID_ARG, "n must be in [0, 65535], got " + std::to_string(n));
  if (n > 0 && (!d_streams || !d_blobs)) return fail(PWPP_ERR_INVALID_ARG, "d_streams and d_blobs must not be NULL when n > 0");
  const int64_t need = (int64_t) pwpp_state_blob_size(ctx);
  if (blob_stride < need || blob_stride % 16 != 0)
    return fail(PWPP_ERR_INVALID_ARG, "blob_stride " + std::to_string(blob_stride) + " must be a multiple of 16 and at least pwpp_state_blob_size = " +
                                          std::to_string(need));
  if (reinterpret_cast<uintptr_t>(d_blobs) % 16 != 0) return fail(PWPP_ERR_INVALID_ARG, "d_blobs must be 16-byte aligned");
  *run = n > 0;
  return PWPP_OK;
}
static StateStore state_store(pwpp_ctx* ctx) {
  return StateStore{ctx->d_states.p, reinterpret_cast<long long*>(ctx->d_hist.p), ctx->hist_stride, ctx->d_stream_hcap.p, ctx->num_streams};
}

int pwpp_export_states_device(pwpp_ctx* ctx, int n, const int32_t* d_streams, void* d_blobs, int64_t blob_stride, int32_t* d_status, void* cuda_stream) {
  bool run = false;
  int rc = check_state_list(ctx, n, d_streams, d_blobs, blob_stride, &run);
  if (rc || !run) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  k_state_export<<<n, SC_THREADS, 0, s>>>(d_streams, state_store(ctx), static_cast<unsigned char*>(d_blobs), blob_stride, d_status);
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  return PWPP_OK;
}

int pwpp_import_states_device(pwpp_ctx* ctx, int n, const int32_t* d_streams, const void* d_blobs, int64_t blob_stride, int32_t* d_status,
                              void* cuda_stream) {
  bool run = false;
  int rc = check_state_list(ctx, n, d_streams, d_blobs, blob_stride, &run);
  if (rc || !run) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  k_state_import_claim<<<(n + SC_CLAIM_THREADS - 1) / SC_CLAIM_THREADS, SC_CLAIM_THREADS, 0, s>>>(n, d_streams, ctx->num_streams, ctx->d_claim.p);
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  k_state_import<<<n, SC_THREADS, 0, s>>>(d_streams, state_store(ctx), static_cast<const unsigned char*>(d_blobs), blob_stride, ctx->d_claim.p, d_status);
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  return PWPP_OK;
}

// bytes from src's buffer on device src_dev to dst's on dst_dev, on stream s of dst_dev
static cudaError_t copy_between(void* dst, int dst_dev, const void* src, int src_dev, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return cudaSuccess;
  if (dst_dev == src_dev) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s);
  return cudaMemcpyPeerAsync(dst, dst_dev, src, src_dev, bytes, s);
}

int pwpp_clone(const pwpp_ctx* src_c, int device, pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  if (!src_c) return fail(PWPP_ERR_INVALID_ARG, "src is NULL");
  pwpp_ctx* src = const_cast<pwpp_ctx*>(src_c);   // fetching the last call's host description caches it; nothing observable changes
  if (any_bound(src)) return fail(PWPP_ERR_INVALID_ARG, "pwpp_clone: the source holds a bound call; pwpp_unbind_call first");
  if (device < 0) device = src->device;
  int rc = bind_device(src);
  if (rc) return rc;
  if (src->last_stream) CU_TRY(cudaStreamSynchronize(src->last_stream));
  CU_TRY(cudaStreamSynchronize(src->stream));
  const int nf = src->last_nframes;
  if (nf > 0) {
    rc = fetch_counts(src);   // the host offsets of a bound call's results (after an unbind) come with the counts
    if (rc) return rc;
  }
  pwpp_ctx* c = nullptr;
  rc = create_impl(src->set_params.data(), src->num_sets, src->stream_set.data(), device, src->num_streams, 0, &c);
  if (rc) return rc;
  auto done = [&](int code) { if (code) pwpp_destroy(c); else *out = c; return code; };
  const int sd = src->device;
  cudaStream_t s = c->stream;
  c->order_mode = src->order_mode;
  c->arith = src->arith;
#define CU_CLONE(expr) do { const cudaError_t _e = (expr); if (_e != cudaSuccess) return done(fail(PWPP_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e))); } while (0)
  // the point capacity of src's per-point buffers
  CU_CLONE(c->d_in.reserve(src->d_in.cap));
  CU_CLONE(c->d_bin_ids.reserve(src->d_bin_ids.cap));
  CU_CLONE(c->d_sorted.reserve(src->d_sorted.cap));
  CU_CLONE(c->d_part.reserve(src->d_part.cap));
  CU_CLONE(c->d_out_idx.reserve(src->d_out_idx.cap));
  const size_t ns = (size_t) src->num_streams;
  CU_CLONE(copy_between(c->d_states.p, device, src->d_states.p, sd, ns * sizeof(StreamState), s));
  CU_CLONE(copy_between(c->d_hist.p, device, src->d_hist.p, sd, ns * 2 * 4 * src->hist_stride * sizeof(double), s));
  if (nf > 0) {
    const long long total = src->last_total;
    const size_t nb = (size_t) src->gs.nbs;
    rc = reserve_work(c, nf, total, 0, true, false);
    if (rc) return done(rc);
    CU_CLONE(copy_between(c->d_counts.p, device, src->d_counts.p, sd, (size_t) 3 * nf * sizeof(int), s));
    CU_CLONE(copy_between(c->d_out_idx.p, device, src->d_out_idx.p, sd, (size_t) total * sizeof(int), s));
    CU_CLONE(copy_between(c->d_in.p, device, src->last_pts, sd, (size_t) total * sizeof(float4), s));
    CU_CLONE(copy_between(c->d_bin_ids.p, device, src->d_bin_ids.p, sd, (size_t) total * sizeof(unsigned short), s));
    CU_CLONE(copy_between(c->d_fits.p, device, src->d_fits.p, sd, nf * nb * sizeof(BinFit), s));
    CU_CLONE(copy_between(c->d_centers.p, device, src->d_centers.p, sd, nf * nb * 3 * sizeof(float), s));
    CU_CLONE(copy_between(c->d_normals.p, device, src->d_normals.p, sd, nf * nb * 3 * sizeof(float), s));
    c->last_nframes = nf;
    c->last_total = total;
    c->pt_off = src->pt_off;
    c->frame_set = src->frame_set;
    c->last_pts = c->d_in.p;
    c->last_stream = s;
  }
  c->last_time_us = src->last_time_us;
  CU_CLONE(cudaStreamSynchronize(s));
#undef CU_CLONE
  return done(PWPP_OK);
}

int pwpp_device_results(pwpp_ctx* ctx, const int32_t** d_indices, const int32_t** d_num_ground) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (d_indices) *d_indices = ctx->d_out_idx.p;
  if (d_num_ground) *d_num_ground = ctx->d_counts.p;
  return PWPP_OK;
}

int pwpp_set_output_order(pwpp_ctx* ctx, int order) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (order != PWPP_ORDER_BIN && order != PWPP_ORDER_REFERENCE && order != PWPP_ORDER_REFERENCE_EXACT)
    return fail(PWPP_ERR_INVALID_ARG, "order must be PWPP_ORDER_BIN, PWPP_ORDER_REFERENCE or PWPP_ORDER_REFERENCE_EXACT");
  if (any_bound(ctx)) return fail(PWPP_ERR_INVALID_ARG, "the output order cannot change while a call is bound (it keeps the order it was bound with)");
  if (order != ctx->order_mode) ++g_alloc_gen;   // captured graphs were recorded with the other launch sequence
  ctx->order_mode = order;
  return PWPP_OK;
}

int pwpp_set_arithmetic(pwpp_ctx* ctx, int arith) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (arith != PWPP_ARITH_DOUBLE && arith != PWPP_ARITH_REFERENCE) return fail(PWPP_ERR_INVALID_ARG, "arith must be PWPP_ARITH_DOUBLE or PWPP_ARITH_REFERENCE");
  if (any_bound(ctx)) return fail(PWPP_ERR_INVALID_ARG, "the arithmetic cannot change while a call is bound (it keeps the arithmetic it was bound with)");
  if (arith != ctx->arith) ++g_alloc_gen;   // captured graphs were recorded with the other fit kernels
  ctx->arith = arith;
  return PWPP_OK;
}

int pwpp_arithmetic(const pwpp_ctx* ctx) { return ctx ? ctx->arith : PWPP_ERR_INVALID_ARG; }

int pwpp_order_exact_counts(pwpp_ctx* ctx, uint64_t out[3], int reset) {
  if (!ctx || !out) return fail(PWPP_ERR_INVALID_ARG, "ctx or out is NULL");
  CU_TRY(cudaSetDevice(ctx->device));
  CU_TRY(cudaDeviceSynchronize());
  unsigned long long c[OX_NUM_STATS];
  CU_TRY(cudaMemcpy(c, ctx->d_ox_counts.p, sizeof c, cudaMemcpyDeviceToHost));
  for (int k = 0; k < OX_NUM_STATS; ++k) out[k] = c[k];
  if (reset) CU_TRY(cudaMemset(ctx->d_ox_counts.p, 0, sizeof c));
  return PWPP_OK;
}

int pwpp_host_results(pwpp_ctx* ctx, const int32_t** h_indices, const int32_t** h_num_ground, const int64_t** h_offsets) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (ctx->last_nframes <= 0) return fail(PWPP_ERR_INVALID_ARG, "no estimate call yet");
  int rc = fetch_indices(ctx);
  if (rc) return rc;
  static_assert(sizeof(long long) == sizeof(int64_t), "offset table type");
  if (h_indices) *h_indices = ctx->h_out_idx.p;
  if (h_num_ground) *h_num_ground = ctx->h_counts.p;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(ctx->pt_off.data());
  return PWPP_OK;
}

int pwpp_bind_host_to_device(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
  for (char* c = bus; *c; ++c) *c = (char) std::tolower((unsigned char) *c);
  std::string base = std::string("/sys/bus/pci/devices/") + bus;
  int node = -1;
  if (FILE* f = std::fopen((base + "/numa_node").c_str(), "r")) { if (std::fscanf(f, "%d", &node) != 1) node = -1; std::fclose(f); }
  if (node < 0) return -1;
  std::string list;
  if (FILE* f = std::fopen(("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist").c_str(), "r")) {
    char buf[4096] = {0};
    if (std::fgets(buf, sizeof buf, f)) list = buf;
    std::fclose(f);
  }
  if (list.empty()) return -1;
  cpu_set_t set;
  CPU_ZERO(&set);
  int ncpu = 0;
  const char* p = list.c_str();
  while (*p) {   // "0-31,64-95"
    char* end = nullptr;
    long a = std::strtol(p, &end, 10);
    if (end == p) break;
    long b = a;
    if (*end == '-') { p = end + 1; b = std::strtol(p, &end, 10); }
    for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int) c, &set); ++ncpu; }
    p = (*end == ',') ? end + 1 : end;
    if (*end != ',' ) break;
  }
  if (ncpu == 0 || sched_setaffinity(0, sizeof set, &set) != 0) return -1;
  return node;
}

int pwpp_copy_bin_results(pwpp_ctx* ctx, int f, pwpp_bin_result* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  if (ctx->sets_on_device && (rc = fetch_offsets(ctx))) return rc;   // the sets the bound call's frames ran with
  rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  const int nb = ctx->gs.g[ctx->frame_set[f]].nbins;   // the records of the frame's set
  CU_TRY(cudaMemcpy(dst, ctx->d_fits.p + (size_t) f * ctx->gs.nbs, (size_t) nb * sizeof(BinFit), cudaMemcpyDeviceToHost));
  return PWPP_OK;
}
int pwpp_copy_bin_ids(pwpp_ctx* ctx, int f, uint16_t* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_offsets(ctx);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  const int n = frame_n(ctx, f);
  if (n > 0) CU_TRY(cudaMemcpy(dst, ctx->d_bin_ids.p + ctx->pt_off[f], (size_t) n * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  return PWPP_OK;
}

#if defined(PWPP_PHASE_CLOCKS)
// diagnostic builds only: cycles thread 0 of the k_fit_group CTAs spent per phase, [3 classes][16]; reset = 1 clears them
int pwpp_debug_phase_clocks(pwpp_ctx* ctx, unsigned long long* out, int reset) {
  if (!ctx) return PWPP_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (out) cudaMemcpyFromSymbol(out, g_phase_clk, sizeof(unsigned long long) * 48);
  if (reset) { static unsigned long long z[48]; cudaMemcpyToSymbol(g_phase_clk, z, sizeof z); }
  return PWPP_OK;
}
int pwpp_debug_events(pwpp_ctx* ctx, unsigned* out, int max_events) {
  if (!ctx) return -1;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (out && max_events >= 16384) cudaMemcpyFromSymbol(out, g_ev, (size_t) 16384 * 16);
  static uint4 z[16384];
  cudaMemcpyToSymbol(g_ev, z, sizeof z);
  return 16384;
}
#endif

}  // extern "C"
